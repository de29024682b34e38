"""jxl_rs_b200 — H100 (sm_90a) VarDCT decode hot path behind the jxl-rs decoder seam.

Only the pieces the path needs live here: `csrc/` (CUDA kernels, C ABI, host
front-end) and the host-side mirror of the reference's decoder interface.
"""
from .abi import JxgError, library_path, load_library  # noqa: F401
from .decoder import (Batch, JxgContext, JxlPixelFormat, LfParsedFrame, ModularBatch, ModularParsedFrame,  # noqa: F401
                      ParsedFrame, PipelinedDecoder, PrefixParsedFrame, bind_to_gpu_numa_node, decode_files,
                      decode_modular_files, decode_prefixes, decode_thumbnails, effective_cpus, gpu_numa_cpus)
