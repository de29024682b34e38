"""Streaming entry point (PipelinedDecoder: parse-ahead pool, dispatcher thread, deferred multi-threaded staging, two
contexts) against plain one-batch decodes, plus large-geometry property checks (BASELINE config 4 shape: one big image,
EPF iters 3, 64x64 transforms)."""
import numpy as np
import pytest

from jxl_rs_b200 import abi

pytestmark = pytest.mark.gpu


def test_pipelined_decoder_matches_single_batches():
    import torch
    import jxl_rs_b200 as j
    import synth
    sets = [[synth.encode_synthetic(520 + 8 * i, 300 + 16 * k, 40 + 10 * k + i, 0.6, 2, 1, 1) for i in range(5)] for k in range(4)]
    ctx = j.JxgContext(0)
    want = [[t.numpy().copy() for t in j.decode_files(ctx, files)] for files in sets]
    ctx.close()
    dec = j.PipelinedDecoder(0, depth=2, staging_threads=3)
    outs = []
    for files in sets:
        bufs = []
        for f in files:
            fr = j.ParsedFrame(f)
            bufs.append(torch.empty((fr.height, fr.width, 3), dtype=torch.uint8).pin_memory())
        outs.append(bufs)
        dec.submit(files, [(b.data_ptr(), b.shape[1] * 3) for b in bufs])
    dec.drain()
    for w, o in zip(want, outs):
        for a, b in zip(w, o):
            assert np.array_equal(a, b.numpy())
    # a corrupt file in a later batch surfaces as an error of drain(), and the decoder stays usable
    bad = bytearray(sets[0][0])
    bad[len(bad) // 2] ^= 0xFF
    dec.submit([bytes(bad)], [(outs[0][0].data_ptr(), outs[0][0].shape[1] * 3)])
    with pytest.raises(abi.JxgError):
        dec.drain()
    dec.submit(sets[1], [(b.data_ptr(), b.shape[1] * 3) for b in outs[1]])
    dec.drain()
    assert np.array_equal(want[1][0], outs[1][0].numpy())
    dec.close()


def test_large_single_image_epf3():
    """8192 x 4096, EPF iters 3, Gaborish, transform profile with the 64x64 family: 512 groups of one image."""
    import torch
    import jxl_rs_b200 as j
    import synth
    from tests import oracle_binding as ob
    w, h = 8192, 4096
    data = synth.encode_synthetic(w, h, 77, 0.8, 3, 1, 2)
    ref, _ = ob.decode_file(data, abi.FORMAT_RGB_U8)
    ctx = j.JxgContext(0)
    (out,) = j.decode_files(ctx, [data])
    ctx.close()
    diff = np.abs(out.numpy().astype(np.int16) - ref.astype(np.int16))
    assert diff.max() <= 1
    assert (diff != 0).mean() < 0.01


def test_device_survives_corrupt_streams(golden_dir):
    """Mutated files that still get through the front-end are decoded on the GPU: every outcome must be a clean result
    or a JxgError — no CUDA fault — and the context must still decode a good file afterwards."""
    import glob
    import os
    import torch
    import jxl_rs_b200 as j
    import synth
    from tests.fuzz_util import mutants
    paths = sorted(glob.glob(os.path.join(golden_dir, "jxl", "*.jxl")))
    if os.environ.get("JXG_TEST_EXPERIMENTAL") != "1":
        # fixtures added with the extra-channel support (see test_gpu_zz_extra_channels.py) join the mutation set once
        # that support has had its first run on a device
        new = {"3x3a_srgb_lossy.jxl", "alpha_premultiplied.jxl", "dice.jxl", "squeeze_alpha.jxl", "upsampled_alpha.jxl"}
        paths = [p for p in paths if os.path.basename(p) not in new]
    ctx = j.JxgContext(0)
    decoded = failed = 0
    for _, data in mutants(paths, seed=99, count=220):
        for parse_cls, modular in ((j.ParsedFrame, False), (j.ModularParsedFrame, True)):
            try:
                fr = parse_cls(data)
            except abi.JxgError:
                continue
            if fr.width * fr.height > 40_000_000:
                continue
            out = torch.empty((fr.height, fr.width, 3), dtype=torch.uint8).pin_memory()
            b = j.ModularBatch(ctx) if modular else j.Batch(ctx, 1)
            try:
                if modular:
                    b.add(fr, out.data_ptr(), fr.width * 3, False)
                else:
                    b.add(fr, out.data_ptr(), fr.width * 3, abi.FORMAT_RGB_U8, False)
                b.run()
                b.wait()
                decoded += 1
            except abi.JxgError as e:
                assert e.code != -20, f"CUDA error on a corrupt stream: {e}"
                failed += 1
            finally:
                b.close()
    assert decoded + failed > 20
    good = synth.encode_synthetic(300, 200, 5, 0.7, 2, 1, 1)
    (o,) = j.decode_files(ctx, [good])
    assert o.shape == (200, 300, 3)
    ctx.close()


def test_c_abi_rejects_inconsistent_descriptors():
    """jxg_batch_add_frame is the boundary a foreign host (the Rust shim) calls: every index-bearing field of the
    descriptor is checked on the host before a kernel can dereference it; a descriptor of the in-tree front-end passes."""
    import ctypes as C
    import torch
    import jxl_rs_b200 as j
    import synth
    data = synth.encode_synthetic(300, 200, 9, 0.5, 2, 1, 1)
    fr = j.ParsedFrame(data)
    ctx = j.JxgContext(0)
    out = torch.empty((200, 300, 3), dtype=torch.uint8, device="cuda:0")

    def try_add(mutate):
        d, hf, off, ln, n = fr.desc(abi.FORMAT_RGB_U8)
        keep = mutate(d)  # noqa: F841 - keeps replacement buffers alive
        b = j.Batch(ctx, 1)
        try:
            b.add_desc(d, hf, off, ln, n, out.data_ptr(), 300 * 3, True)
            return 0
        except abi.JxgError as e:
            return e.code
        finally:
            b.close()

    assert try_add(lambda d: None) == 0

    def bad_context_map(d):
        p = d.passes[0]
        buf = (C.c_uint8 * p.num_contexts).from_buffer_copy(C.string_at(p.context_map, p.num_contexts))
        buf[5] = 255
        p.context_map = C.cast(buf, C.c_void_p)
        return buf

    def bad_transform(d):
        nb = ((300 + 7) // 8) * ((200 + 7) // 8)
        buf = (C.c_uint8 * nb).from_buffer_copy(C.string_at(d.transform_map, nb))
        buf[nb - 1] = 128 | 24  # a 256x256 varblock starting in the last block: crosses the frame
        d.transform_map = C.cast(buf, C.c_void_p)
        return buf

    def bad_quant_lf(d):
        nb = ((300 + 7) // 8) * ((200 + 7) // 8)
        buf = (C.c_uint8 * nb)(*([200] * nb))
        d.quant_lf = C.cast(buf, C.c_void_p)
        return buf

    def setter(name, value):
        def f(d):
            setattr(d, name, value)
        return f

    for mutate in (bad_context_map, bad_transform, bad_quant_lf, setter("block_ctx_map_len", 7), setter("num_block_contexts", 200),
                   setter("orientation", 9), setter("output_tf", 77), setter("global_scale", 0)):
        assert try_add(mutate) == -22, mutate  # JXG_ERR_ARGUMENT
    ctx.close()


def test_c_abi_rejects_unknown_debug_stages():
    """Debug stops 0-2 and XYB tap stage 0 are the only stages there are: a NULL batch or any other stage is
    JXG_ERR_ARGUMENT, and stage 0 of a run stopped after the transforms still reads."""
    import torch
    import jxl_rs_b200 as j
    import synth
    fr = j.ParsedFrame(synth.encode_synthetic(300, 200, 9, 0.5, 2, 1, 1))
    ctx = j.JxgContext(0)
    out = torch.empty((3, 200, 300), dtype=torch.float32).pin_memory()
    b = j.Batch(ctx, 1)
    try:
        lib = b._lib
        assert lib.jxg_batch_set_debug_stop(None, 2) == -22  # JXG_ERR_ARGUMENT
        for stage in (-1, 3, 4):
            assert lib.jxg_batch_set_debug_stop(b._h, stage) == -22, stage
        assert lib.jxg_batch_set_debug_stop(b._h, 2) == 0
        b.add(fr, out.data_ptr(), 300 * 4, abi.FORMAT_XYB_F32_PLANAR, False)
        b.run()
        b.wait()
        assert np.isfinite(b.read_xyb(0, 0)).all()
        for stage in (1, 2):
            with pytest.raises(abi.JxgError):
                b.read_xyb(0, stage)
    finally:
        b.close()
        ctx.close()
