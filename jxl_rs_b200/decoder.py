"""Host-side mirror of the jxl-rs decoder API for the VarDCT hot path.

Reference shape (jxl/src/api/decoder.rs:33-266, data_types.rs:154, image/output_buffer.rs:26):
    JxlDecoder::process(input, buffers, runner)  ->  pixels in JxlOutputBuffer
Here a *batch* of frames is decoded per call (one crossing of the host/device
boundary per batch, SURVEY §3.5). PyTorch supplies device memory, pinned host
memory and streams only; all compute is in libjxgpu.so.
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import abi


@dataclass
class JxlPixelFormat:
    """jxl/src/api/data_types.rs:154 (colour part only)."""
    color_type: str = "RGB"          # "RGB" | "RGBA"
    data_format: str = "U8"          # "U8" | "U16" | "F16" | "F32" (JxlDataFormat, 16-bit samples in native endianness)

    def abi_format(self):
        if self.data_format == "U8":
            return abi.FORMAT_RGBA_U8 if self.color_type == "RGBA" else abi.FORMAT_RGB_U8
        if self.color_type == "RGB" and self.data_format in ("F32", "U16", "F16"):
            return {"F32": abi.FORMAT_RGB_F32, "U16": abi.FORMAT_RGB_U16, "F16": abi.FORMAT_RGB_F16}[self.data_format]
        raise ValueError(f"unsupported pixel format {self}")


class ParsedFrame:
    """A .jxl file run through the host front-end (headers, TOC, LfGlobal, LF
    groups, HfGlobal): what a Rust host has in `Frame` when it reaches
    decode_and_render_hf_groups (frame/render.rs:143)."""

    def __init__(self, data: bytes, threads: int = 1):
        """threads > 1: the frame's LF groups are decoded on that many host threads (one large image); batches of
        many frames keep 1 and parse frames in parallel instead."""
        self._lib = abi.load_library()
        self._h = C.c_void_p()
        self.info = abi.JxgImageInfo()
        abi.check(self._lib, self._lib.jxg_parse_file_mt(data, len(data), int(threads), C.byref(self._h),
                                                          C.byref(self.info)))

    @property
    def width(self):
        """Output (display-orientation) width: what the caller's buffer must hold."""
        return self.info.width

    @property
    def height(self):
        return self.info.height

    def desc(self, output_format):
        d = abi.JxgFrameDesc()
        hf, off, ln, n = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_uint32()
        abi.check(self._lib, self._lib.jxg_parsed_desc(self._h, output_format, C.byref(d), C.byref(hf), C.byref(off),
                                                       C.byref(ln), C.byref(n)))
        return d, hf, off, ln, n.value

    def region_desc(self, output_format, region):
        """The sub-frame a region (x, y, w, h in output coordinates) decodes (jxg_parsed_region_desc): (desc, hf, off,
        len, n_sections, origin, window); origin is the sub-frame's coded top-left, window the region's top-left in
        the sub-frame's display-oriented output. Valid until the next call on this frame."""
        d = abi.JxgFrameDesc()
        hf, off, ln, n = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_uint32()
        origin, window = (C.c_uint32 * 2)(), (C.c_uint32 * 2)()
        abi.check(self._lib, self._lib.jxg_parsed_region_desc(self._h, output_format, C.byref(_region(region)), C.byref(d),
                                                              C.byref(hf), C.byref(off), C.byref(ln), C.byref(n),
                                                              origin, window))
        return d, hf, off, ln, n.value, tuple(origin), tuple(window)

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.jxg_parsed_free(self._h)
            self._h = C.c_void_p()


class PrefixParsedFrame(ParsedFrame):
    """A prefix of a VarDCT .jxl file (jxg_parse_file_prefix): a bare codestream cut anywhere after HfGlobal. Usable
    with Batch.add, whole or with a region: each HF group is decoded from the passes of it that have arrived, and a
    group with none shows the LF image upsampled 8x. A complete prefix decodes as ParsedFrame does."""

    def __init__(self, data: bytes):
        self._lib = abi.load_library()
        self._h = C.c_void_p()
        self.info = abi.JxgImageInfo()
        abi.check(self._lib, self._lib.jxg_parse_file_prefix(data, len(data), C.byref(self._h), C.byref(self.info)))

    @property
    def passes(self):
        """k_g of each HF group (jxg_parsed_group_passes): the passes it is decoded with, 0 = LF upsampled 8x."""
        out = np.zeros(self.info.num_groups, np.uint8)
        abi.check(self._lib, self._lib.jxg_parsed_group_passes(self._h, out.ctypes.data, out.size))
        return out

    def region_plan(self, region):
        """The groups a region (x, y, w, h in output coordinates) decodes (jxg_parsed_prefix_region_plan), no device
        needed: (groups, passes, lf_window) with groups their whole-frame indices in sub-frame order, passes their k_g,
        and lf_window the LF rectangle (x0, y0, x1, y1) uploaded for the upsampling, (0, 0, 0, 0) when none is."""
        reg = C.byref(_region(region))
        n = C.c_uint32()
        abi.check(self._lib, self._lib.jxg_parsed_prefix_region_plan(self._h, reg, None, None, 0, C.byref(n), None))
        groups, passes = np.zeros(n.value, np.uint32), np.zeros(n.value, np.uint8)
        win = (C.c_uint32 * 4)()
        abi.check(self._lib, self._lib.jxg_parsed_prefix_region_plan(self._h, reg, groups.ctypes.data, passes.ctypes.data,
                                                                     n.value, C.byref(n), win))
        return groups, passes, tuple(win)


def _region(region):
    x, y, w, h = (int(v) for v in region)
    return abi.JxgRegion(x, y, w, h)


def _out_size(frame, region):
    """(height, width) of the output of a frame, or of a region (x, y, w, h) of it."""
    return (frame.height, frame.width) if region is None else (int(region[3]), int(region[2]))


class JxgContext:
    """One per GPU / rank (jxg_init)."""

    def __init__(self, device: int = 0):
        self._lib = abi.load_library()
        self._h = C.c_void_p()
        abi.check(self._lib, self._lib.jxg_init(device, C.byref(self._h)))
        self.device = device

    def set_pool_fill(self, byte: int):
        """Test hook (jxg_context_set_pool_fill): with `byte` in 0..255 every later batch run writes it over the
        context's device pools and staging arena first, so that outputs cannot depend on what earlier batches left
        there; -1 (the default) turns it off. Each begin, run and rerun uses the byte in force when it is called."""
        abi.check(self._lib, self._lib.jxg_context_set_pool_fill(self._h, int(byte)))

    def set_sm_budget(self, n: int):
        """Test hook (jxg_context_set_sm_budget): with n >= 1 the context's later batches are scheduled as if the device
        had n SMs (entropy lanes per warp and per frame, queued streams, Modular grids); 0 (the default) uses the
        device's own count. Outputs do not depend on it."""
        abi.check(self._lib, self._lib.jxg_context_set_sm_budget(self._h, int(n)))

    def close(self):
        if self._h.value:
            self._lib.jxg_shutdown(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _BatchHandle:
    """The handle of either batch kind (C functions `<_PREFIX>begin / run / rerun_device / end`): one live batch per
    context; run and rerun_device take a raw cudaStream_t, 0 for the context's own stream."""
    _PREFIX = ""

    def __init__(self, ctx: JxgContext, *begin_args):
        self._lib = ctx._lib
        self._ctx = ctx
        self._h = C.c_void_p()
        abi.check(self._lib, getattr(self._lib, self._PREFIX + "begin")(ctx._h, *begin_args, C.byref(self._h)))

    def run(self, stream_ptr: int = 0):
        abi.check(self._lib, getattr(self._lib, self._PREFIX + "run")(self._h, C.c_void_p(stream_ptr)))

    def rerun_device(self, stream_ptr: int = 0):
        abi.check(self._lib, getattr(self._lib, self._PREFIX + "rerun_device")(self._h, C.c_void_p(stream_ptr)))

    def close(self):
        if self._h.value:
            if self._ctx._h.value:  # a batch that outlives its context is abandoned, not freed through it
                getattr(self._lib, self._PREFIX + "end")(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Batch(_BatchHandle):
    """jxg_batch_*: frames decoded together by one kernel pipeline."""
    _PREFIX = "jxg_batch_"

    def __init__(self, ctx: JxgContext, n_hint: int = 0, staging_threads: int = 0):
        """staging_threads > 0: large input copies are deferred to run() and done by that many host threads
        (jxg_batch_set_deferred_copy); the ParsedFrames added are kept alive by this object."""
        super().__init__(ctx, n_hint)
        self._keep = []
        self.frames = []
        if staging_threads > 0:
            abi.check(self._lib, self._lib.jxg_batch_set_deferred_copy(self._h, staging_threads))

    def add(self, frame: ParsedFrame, out_ptr: int, row_stride: int, fmt: int, out_is_device: bool, region=None):
        """region: None for the whole frame, or (x, y, w, h) in output coordinates: only that rectangle is decoded
        and stored, into a buffer of h rows of w pixels (jxg_batch_add_parsed_region)."""
        dev = 1 if out_is_device else 0
        if region is None:
            abi.check(self._lib, self._lib.jxg_batch_add_parsed(self._h, frame._h, fmt, C.c_void_p(out_ptr), row_stride, dev))
        else:
            abi.check(self._lib, self._lib.jxg_batch_add_parsed_region(self._h, frame._h, fmt, C.byref(_region(region)),
                                                                       C.c_void_p(out_ptr), row_stride, dev))
        self.frames.append(frame)

    def add_desc(self, desc, hf, off, ln, n, out_ptr, row_stride, out_is_device):
        abi.check(self._lib, self._lib.jxg_batch_add_frame(self._h, C.byref(desc), hf, off, ln, n, C.c_void_p(out_ptr),
                                                           row_stride, 1 if out_is_device else 0))

    def set_debug_stop(self, stage: int):
        self._lib.jxg_batch_set_debug_stop(self._h, stage)

    STAGES = ["memset", "entropy", "dequant_idct", "gaborish", "epf0", "epf1", "epf2", "xyb_store"]

    def set_profile(self, on: bool):
        abi.check(self._lib, self._lib.jxg_batch_set_profile(self._h, 1 if on else 0))

    def stage_times(self):
        ms = (C.c_float * 8)()
        abi.check(self._lib, self._lib.jxg_batch_stage_times(self._h, ms, 8))
        return dict(zip(self.STAGES, [float(v) for v in ms]))

    def stage_marks(self):
        """Absolute device times (ms) of the 9 stage events of the last run, then of the run's first event (before the
        H2D copy) and its last one (behind the D2H copies) (jxg_batch_stage_marks)."""
        ms = (C.c_float * 11)()
        abi.check(self._lib, self._lib.jxg_batch_stage_marks(self._h, ms, 11))
        return [float(v) for v in ms]

    def wait(self):
        f, g = C.c_uint32(), C.c_uint32()
        abi.check(self._lib, self._lib.jxg_batch_wait(self._h, C.byref(f), C.byref(g)))

    def stats(self):
        k, h, d, ms = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_float()
        self._lib.jxg_batch_stats(self._h, C.byref(k), C.byref(h), C.byref(d), C.byref(ms))
        return {"kernel_launches": k.value, "h2d_bytes": h.value, "d2h_bytes": d.value, "device_ms": ms.value}

    def entropy_stats(self):
        """Which entropy kernel instances decode this batch (jxg_batch_entropy_stats): stream counts of k_entropy_lean,
        k_entropy_fast and k_entropy, the lean kernel's (4, 2, 0) and shared-memory context map forms, and its lanes
        per warp (0 before run() or without lean streams)."""
        nl, nf, ns, s = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        a420, smem = C.c_int(), C.c_int()
        abi.check(self._lib, self._lib.jxg_batch_entropy_stats(self._h, C.byref(nl), C.byref(nf), C.byref(ns),
                                                               C.byref(a420), C.byref(smem), C.byref(s)))
        return {"lean": nl.value, "fast": nf.value, "slow": ns.value, "lean_all_420": bool(a420.value),
                "lean_ctx_smem": bool(smem.value), "lean_S": s.value}

    def entropy_schedule(self):
        """The entropy schedule of the last run() (jxg_batch_entropy_schedule): the lean kernel's lanes per warp
        ("lean_S", 0 without lean streams) and grid ("lean_ctas"), the fast kernel's streams per warp ("fast_S", 0
        without such streams), and per frame ("frames") a dict of its lean streams ("count"), the lanes that start on
        them ("lanes"; the rest are queued), its CTAs ("ctas") and the pulls of its lanes from its stream queue
        ("pulls": "count" when every queued stream was taken once). Waits for the run."""
        def one(f):
            v = [C.c_uint32() for _ in range(5)]
            abi.check(self._lib, self._lib.jxg_batch_entropy_schedule(self._h, f, *(C.byref(x) for x in v)))
            return [x.value for x in v]
        count, lanes, ctas, fast_s, pulls = one(abi.ALL_FRAMES)
        frames = []
        for f in range(len(self.frames)):
            c, la, ct, _, p = one(f)
            frames.append({"count": c, "lanes": la, "ctas": ct, "pulls": p})
        return {"lean_S": self.entropy_stats()["lean_S"], "lean_count": count, "lean_lanes": lanes, "lean_ctas": ctas,
                "fast_S": fast_s, "lean_pulls": pulls, "frames": frames}

    def stream_status(self, f: int):
        """Status word of each group of whole frame f after wait() (jxg_batch_stream_status): 0 or a JXG_ERR_* code."""
        n = self.frames[f].info.num_groups
        out = np.empty(n, np.int32)
        abi.check(self._lib, self._lib.jxg_batch_stream_status(self._h, f, out.ctypes.data_as(C.POINTER(C.c_int32)), n))
        return out

    def transform_plan(self, f: int, num_groups: int = 0):
        """Transform-class partition of the block plan of whole frame f (jxg_batch_read_transform_plan): counts
        [groups, 8] u32 (classes 0..4, then zeros) and the varblock entries [groups, 1024] u32 (ordinal | bx << 10 |
        by << 15 | transform type << 20), class after class.
        num_groups: the frame's group count, needed for frames added with add_desc."""
        n = num_groups or self.frames[f].info.num_groups
        counts = np.zeros((n, 8), np.uint32)
        seqs = np.zeros((n, 1024), np.uint32)
        abi.check(self._lib, self._lib.jxg_batch_read_transform_plan(self._h, f, counts.ctypes.data, seqs.ctypes.data, n))
        return counts, seqs

    def read_coeffs(self, f: int):
        n = self.frames[f].info.num_groups * 3 * 65536
        out = np.empty(n, np.int32)
        abi.check(self._lib, self._lib.jxg_batch_read_coeffs(self._h, f, out.ctypes.data_as(C.c_void_p), n))
        return out.reshape(self.frames[f].info.num_groups, 3, 65536)

    def read_xyb(self, f: int, stage: int):
        w, h = self.frames[f].info.coded_width, self.frames[f].info.coded_height
        ps, pr = (w + 7) // 8 * 8, (h + 7) // 8 * 8
        out = np.empty(3 * ps * pr, np.float32)
        abi.check(self._lib, self._lib.jxg_batch_read_xyb(self._h, f, stage, out.ctypes.data_as(C.c_void_p), out.size))
        return out.reshape(3, pr, ps)


def decode_files(ctx: JxgContext, files, pixel_format: JxlPixelFormat = JxlPixelFormat(), to_host: bool = True,
                 regions=None):
    """Decodes a list of .jxl byte strings; returns a list of torch tensors
    (H x W x C). Host results land in pinned memory (JxlOutputBuffer analogue).
    regions: None, or one entry per file: None (the whole image) or (x, y, w, h) in output coordinates, which decodes
    only that rectangle into an h x w x C tensor."""
    import torch
    fmt = pixel_format.abi_format()
    cpus = effective_cpus()
    per_file = max(1, cpus // max(1, len(files)))
    if len(files) > 1:
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=min(cpus, len(files))) as ex:
            frames = list(ex.map(lambda f: ParsedFrame(f, per_file), files))
    else:
        frames = [ParsedFrame(f, per_file) for f in files]
    if regions is None:
        regions = [None] * len(frames)
    if len(regions) != len(frames):
        raise ValueError("regions: one entry per file")
    batch = Batch(ctx, len(frames))
    outs = []
    try:  # a corrupt frame must not leave the context with a live batch
        for fr, reg in zip(frames, regions):
            ch = 4 if fmt == abi.FORMAT_RGBA_U8 else 3
            dt = {abi.FORMAT_RGB_F32: torch.float32, abi.FORMAT_RGB_U16: torch.uint16, abi.FORMAT_RGB_F16: torch.float16}.get(fmt, torch.uint8)
            h, w = _out_size(fr, reg)
            if to_host:
                t = torch.empty((h, w, ch), dtype=dt).pin_memory()
            else:
                t = torch.empty((h, w, ch), dtype=dt, device=f"cuda:{ctx.device}")
            outs.append(t)
            batch.add(fr, t.data_ptr(), w * ch * t.element_size(), fmt, not to_host, reg)
        batch.run()
        batch.wait()
    finally:
        batch.close()
    return outs


def _parse_cpulist(text):
    cpus = set()
    for part in text.strip().split(","):
        if not part:
            continue
        lo, _, hi = part.partition("-")
        cpus.update(range(int(lo), int(hi or lo) + 1))
    return cpus


def gpu_numa_cpus(device: int, sysfs: str = "/sys"):
    """(numa_node, set of CPUs) of the NUMA node the GPU's PCIe root hangs off, or (None, None) when the platform does
    not say (single-node hosts report -1)."""
    import os
    lib = abi.load_library()
    buf = C.create_string_buffer(32)
    if lib.jxg_device_pci_bus_id(device, buf, 32) != 0:
        return None, None
    try:
        node = int(open(os.path.join(sysfs, "bus/pci/devices", buf.value.decode(), "numa_node")).read())
        if node < 0:
            return None, None
        return node, _parse_cpulist(open(os.path.join(sysfs, f"devices/system/node/node{node}/cpulist")).read())
    except (OSError, ValueError):
        return None, None


def bind_to_gpu_numa_node(device: int):
    """Restricts the calling thread (and every thread it starts afterwards: worker pools, the dispatcher) to the
    CPUs of the GPU's NUMA node. Call it before the pools and the pinned buffers are created: pinned pages are
    allocated on the node of the thread that asks for them, and H2D / D2H copies through a remote node cross the
    inter-socket link (the end-to-end scaling collapse of round 1 at 8 GPUs). Returns a description for logs."""
    import os
    node, cpus = gpu_numa_cpus(device)
    if not cpus:
        return {"numa_node": None, "bound": False}
    try:
        allowed = os.sched_getaffinity(0)
        want = cpus & allowed
        if want:
            os.sched_setaffinity(0, want)
            return {"numa_node": node, "bound": True, "cpus": len(want)}
    except (AttributeError, OSError):
        pass
    return {"numa_node": node, "bound": False}


def effective_cpus() -> int:
    """Host threads this process can really run at once: min(cpu_count, affinity mask, cgroup v2/v1 CPU quota)."""
    import math
    import os
    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except (AttributeError, OSError):
        pass
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if quota != "max":
            n = min(n, max(1, math.ceil(int(quota) / int(period))))
    except (OSError, ValueError):
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            p = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0 and p > 0:
                n = min(n, max(1, math.ceil(q / p)))
        except (OSError, ValueError):
            pass
    return max(1, n)


class PipelinedDecoder:
    """Streaming decode of many batches. `submit()` only queues a batch: its files start parsing on the worker
    pool at once (so parsing of batch k+1.. overlaps everything else) and a dispatcher thread stages each batch
    (parallel copies into the pinned blob), launches it on one of `depth` contexts (own CUDA stream, staging
    arena and device pools, used round-robin) and retires the oldest one when all contexts are busy. Host
    front-end work of batch k+1 therefore overlaps the kernels and the D2H copies of batch k; the output copies of
    all contexts leave on the device's one first-in-first-out D2H stream, so batches retire in launch order.
    This is the serving-shaped entry point (many independent images in flight). bench.py runs it with depth 5."""

    def __init__(self, device: int = 0, depth: int = 3, workers: int = 0, staging_threads: int = 4, parse_ahead: int = 2):
        import os
        import queue
        import threading
        from collections import deque
        from concurrent.futures import ThreadPoolExecutor
        self.ctxs = [JxgContext(device) for _ in range(depth)]
        self.depth = depth
        self.staging_threads = staging_threads
        self.workers = workers or min(64, effective_cpus())
        self.pool = ThreadPoolExecutor(max_workers=self.workers)
        self.inflight = deque()
        self.k = 0
        self.last_stats = {"h2d_bytes": 0, "d2h_bytes": 0, "kernel_launches": 0}
        self._jobs = queue.Queue()
        self._ahead = threading.Semaphore(depth + parse_ahead)  # bounds parsed-but-not-yet-launched batches
        self._error = None
        self.trace = None  # set to [] to record the dispatcher timeline
        self.retire_trace = []  # with trace on: (start, seconds in wait / stats / close) of every retired batch
        self.marks = None  # set to [] to record the device timeline of every batch (stage event times)
        self.marks_ref_host = None  # time.perf_counter() at the device timeline's zero (set with the first marks)
        self._thread = threading.Thread(target=self._dispatch, daemon=True)
        self._thread.start()

    def _retire(self):
        import time
        b = self.inflight.popleft()
        t0 = time.perf_counter()
        try:
            b.wait()
            t1 = time.perf_counter()
            self.last_stats = b.stats()
            if self.marks is not None:
                tcall = time.perf_counter()
                self.marks.append(b.stage_marks())
                if self.marks_ref_host is None:  # the library's reference event was recorded inside that first call
                    self.marks_ref_host = tcall
        finally:
            t2 = time.perf_counter()
            b.close()
        if self.trace is not None:  # ("retire", start, event wait, stats + marks, close)
            self.retire_trace.append((t0, t1 - t0, t2 - t1, time.perf_counter() - t2))

    def _launch(self, futs, outs, fmt, out_is_device, regions):
        import time
        t0 = time.perf_counter()
        if len(self.inflight) == self.depth:
            self._retire()
        t1 = time.perf_counter()
        ctx = self.ctxs[self.k % self.depth]
        self.k += 1
        b = Batch(ctx, len(futs), self.staging_threads)
        if self.marks is not None:
            b.set_profile(True)
        try:
            frames = [fut.result() for fut in futs]
            t2 = time.perf_counter()
            for fr, (ptr, stride), reg in zip(frames, outs, regions):
                if reg is None:  # the five-argument call whole frames always made (stand-in batches implement only it)
                    b.add(fr, ptr, stride, fmt, out_is_device)
                else:
                    b.add(fr, ptr, stride, fmt, out_is_device, reg)
            t3 = time.perf_counter()
            b.run()
        except Exception:
            b.close()
            raise
        self.inflight.append(b)
        if self.trace is not None:  # host-side timeline of the dispatcher (seconds): start, retire, parse wait, add, run
            self.trace.append((t0, t1 - t0, t2 - t1, t3 - t2, time.perf_counter() - t3))

    def _dispatch(self):
        while True:
            job = self._jobs.get()
            try:
                if job is None:
                    return
                if isinstance(job, tuple) and job[0] == "drain":
                    try:
                        while self.inflight:
                            self._retire()
                    except Exception as e:  # noqa: BLE001 - reported to the caller of drain()
                        self._error = self._error or e
                    job[1].set()
                    continue
                try:
                    if self._error is None:
                        self._launch(*job)
                except Exception as e:  # noqa: BLE001
                    self._error = self._error or e
                finally:
                    self._ahead.release()
            finally:
                self._jobs.task_done()

    def submit(self, files, outs, fmt: int = abi.FORMAT_RGB_U8, out_is_device: bool = False, regions=None):
        """files: list of .jxl byte strings; outs: list of (data_ptr, row_stride). Returns once the batch is
        queued; its outputs are complete after drain() (or once `depth` later batches have been launched).
        regions: None, or one entry per file: None (the whole image) or (x, y, w, h), the output rectangle that is
        decoded into that file's buffer."""
        regions = [None] * len(files) if regions is None else list(regions)
        if len(regions) != len(files):
            raise ValueError("regions: one entry per file")
        self._ahead.acquire()
        # fewer files than workers (one large image): the spare workers decode LF groups inside each file
        per_file = max(1, self.workers // max(1, len(files)))
        futs = [self.pool.submit(ParsedFrame, f, per_file) for f in files]
        self._jobs.put((futs, list(outs), fmt, out_is_device, regions))

    def drain(self):
        import threading
        ev = threading.Event()
        self._jobs.put(("drain", ev))
        ev.wait()
        if self._error is not None:
            e, self._error = self._error, None
            raise e

    def decode(self, files, outs, fmt: int = abi.FORMAT_RGB_U8, out_is_device: bool = False, regions=None):
        self.submit(files, outs, fmt, out_is_device, regions)
        self.drain()

    def close(self):
        try:
            self.drain()
        finally:
            self._jobs.put(None)
            self._thread.join()
            self.pool.shutdown()
            for c in self.ctxs:
                c.close()


class ModularParsedFrame:
    """A Modular-encoded .jxl file run through the host front-end (headers, TOC, LfGlobal with the global MA tree,
    section 0, ModularLF streams, group headers): the state a Rust host holds when it reaches the ModularHF groups."""

    def __init__(self, data: bytes):
        self._lib = abi.load_library()
        self._h = C.c_void_p()
        self.info = abi.JxgImageInfo()
        abi.check(self._lib, self._lib.jxg_modular_parse_file(data, len(data), C.byref(self._h), C.byref(self.info)))

    @property
    def width(self):
        return self.info.width

    @property
    def height(self):
        return self.info.height

    def colour(self, output_format=abi.FORMAT_RGB_U8):
        """jxg_modular_parsed_colour: {"xyb": bool, "colour_channels": coded colour channels, "lf_quant": the
        LfQuantFactors (X, Y, B) of an XYB frame, "desc": the JxgFrameDesc with the output stage a batch applies for
        `output_format`} (lf_quant and desc are None for a lossless frame)."""
        xyb, nc = C.c_int(), C.c_uint32()
        q = (C.c_float * 3)()
        d = abi.JxgFrameDesc()
        abi.check(self._lib, self._lib.jxg_modular_parsed_colour(self._h, output_format, C.byref(xyb), C.byref(nc), q,
                                                                 C.byref(d)))
        return {"xyb": bool(xyb.value), "colour_channels": nc.value, "lf_quant": tuple(q) if xyb.value else None,
                "desc": d if xyb.value else None}

    def region_plan(self, region):
        """The dependency cone of a region (x, y, w, h in output coordinates; jxg_modular_parsed_region_plan), no device
        needed: (groups, arena, need) with groups the whole-frame indices of the group streams decoded, and per buffer
        of the inverse plan the rectangle the plane memory holds and the one the region needs, as (x0, y0, x1, y1)
        half-open, (0, 0, 0, 0) when empty."""
        reg = C.byref(_region(region))
        ng, nb = C.c_uint32(), C.c_uint32()
        abi.check(self._lib, self._lib.jxg_modular_parsed_region_plan(self._h, reg, None, 0, C.byref(ng), None, 0,
                                                                      C.byref(nb)))
        groups = (C.c_uint32 * max(ng.value, 1))()
        rects = (C.c_uint32 * max(8 * nb.value, 1))()
        abi.check(self._lib, self._lib.jxg_modular_parsed_region_plan(self._h, reg, groups, ng.value, C.byref(ng), rects,
                                                                      nb.value, C.byref(nb)))
        r = [tuple(rects[i * 8:i * 8 + 8]) for i in range(nb.value)]
        return list(groups[:ng.value]), [t[:4] for t in r], [t[4:] for t in r]

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.jxg_modular_parsed_free(self._h)
            self._h = C.c_void_p()


class LfParsedFrame:
    """A VarDCT .jxl file parsed for its 1:8 thumbnail (jxg_lf_parse_file): headers, TOC, LfGlobal and the headers of
    the LF-group streams, nothing of HfGlobal or the HF sections. `info` is what ParsedFrame gives for the same file;
    width / height are the thumbnail's (display orientation)."""

    def __init__(self, data: bytes):
        self._lib = abi.load_library()
        self._h = C.c_void_p()
        self.info = abi.JxgImageInfo()
        abi.check(self._lib, self._lib.jxg_lf_parse_file(data, len(data), C.byref(self._h), C.byref(self.info)))

    @property
    def coded_width(self):
        """Thumbnail width in the coded orientation (the LF image's blocks across)."""
        return (self.info.coded_width + 7) // 8

    @property
    def coded_height(self):
        return (self.info.coded_height + 7) // 8

    @property
    def width(self):
        return (self.info.width + 7) // 8

    @property
    def height(self):
        return (self.info.height + 7) // 8

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.jxg_lf_parsed_free(self._h)
            self._h = C.c_void_p()


class ModularBatch(_BatchHandle):
    """jxg_modular_batch_*: Modular frames whose group streams are decoded together on the GPU."""
    _PREFIX = "jxg_modular_batch_"

    def __init__(self, ctx: JxgContext, lanes_per_warp: int = 1):
        super().__init__(ctx)
        abi.check(self._lib, self._lib.jxg_modular_batch_set_lanes(self._h, lanes_per_warp))
        self.frames = []

    def add(self, frame: ModularParsedFrame, out_ptr: int, row_stride: int, out_is_device: bool, region=None, fmt=None):
        """region: None for the whole frame, or (x, y, w, h) in output coordinates: only what that rectangle depends on
        is decoded, and only it is stored, into a buffer of h rows of w pixels (jxg_modular_batch_add_region).
        fmt: None (RGB u8), or a FORMAT_* of abi (jxg_modular_batch_add_output): any format for an XYB frame, RGB_U8
        for a lossless one."""
        dev = 1 if out_is_device else 0
        if fmt is not None:
            reg = None if region is None else C.byref(_region(region))
            abi.check(self._lib, self._lib.jxg_modular_batch_add_output(self._h, frame._h, fmt, reg, C.c_void_p(out_ptr),
                                                                        row_stride, dev))
        elif region is None:
            abi.check(self._lib, self._lib.jxg_modular_batch_add(self._h, frame._h, C.c_void_p(out_ptr), row_stride, dev))
        else:
            abi.check(self._lib, self._lib.jxg_modular_batch_add_region(self._h, frame._h, C.byref(_region(region)),
                                                                        C.c_void_p(out_ptr), row_stride, dev))
        self.frames.append(frame)

    def add_lf(self, frame: LfParsedFrame, out_ptr: int, row_stride: int, fmt: int, out_is_device: bool):
        """Adds the 1:8 thumbnail of a VarDCT frame (jxg_modular_batch_add_lf) in output format `fmt`."""
        abi.check(self._lib, self._lib.jxg_modular_batch_add_lf(self._h, frame._h, fmt, C.c_void_p(out_ptr), row_stride,
                                                                1 if out_is_device else 0))
        self.frames.append(frame)

    def wait(self):
        """Raises the first failing stream's error; `last_failure` holds its (frame, group), the group being the LF-group
        index for a thumbnail."""
        bf, bg = C.c_uint32(), C.c_uint32()
        r = self._lib.jxg_modular_batch_wait(self._h, C.byref(bf), C.byref(bg))
        self.last_failure = (bf.value, bg.value) if r != abi.JXG_OK else None
        abi.check(self._lib, r)

    def stats(self):
        h2d, d2h, launches = C.c_uint64(), C.c_uint64(), C.c_uint64()
        ms = (C.c_float * 2)()
        abi.check(self._lib, self._lib.jxg_modular_batch_stats(self._h, C.byref(h2d), C.byref(d2h), C.byref(launches), ms))
        return {"h2d_bytes": h2d.value, "d2h_bytes": d2h.value, "kernel_launches": launches.value, "device_ms": ms[0],
                "decode_ms": ms[1]}

    def lz77_stats(self):
        """Group streams of the added frames that use LZ77, those of them in run-length form (every copy at distance 1),
        and the device bytes of their symbol windows."""
        n, rle, win = C.c_uint32(), C.c_uint32(), C.c_uint64()
        abi.check(self._lib, self._lib.jxg_modular_batch_lz77_stats(self._h, C.byref(n), C.byref(rle), C.byref(win)))
        return {"lz77_streams": n.value, "rle_streams": rle.value, "window_bytes": win.value}

    def walk_stats(self):
        """Non-empty group-stream rects of the added frames by the channel walk they take on the device: "generic" (the
        tree walk), "single_leaf" (the table walk of a tree left with one leaf), "by_property" {p: rects} (the table
        walk over property p, 2..15; properties without rects left out) and "table_wp" (table rects whose stream uses
        the weighted predictor)."""
        gen, single, wp = C.c_uint32(), C.c_uint32(), C.c_uint32()
        by = (C.c_uint32 * 16)()
        abi.check(self._lib, self._lib.jxg_modular_batch_walk_stats(self._h, C.byref(gen), C.byref(single), by,
                                                                    C.byref(wp)))
        return {"generic": gen.value, "single_leaf": single.value,
                "by_property": {p: by[p] for p in range(16) if by[p]}, "table_wp": wp.value}

    def read_planes(self, f: int):
        import numpy as np
        fr = self.frames[f]
        out = np.zeros((3, fr.info.coded_height, fr.info.coded_width), np.int32)
        abi.check(self._lib, self._lib.jxg_modular_batch_read_planes(self._h, f, out.ctypes.data, out.size))
        return out


def decode_modular_files(ctx: JxgContext, files, to_host: bool = True, lanes_per_warp: int = 1,
                         pixel_format: JxlPixelFormat = JxlPixelFormat()):
    """Decodes a list of Modular .jxl byte strings on the GPU; returns H x W x C torch tensors of the display-oriented
    images in `pixel_format`. Lossless frames take the default RGB U8 only; XYB (lossy) frames take every format."""
    import torch
    fmt = pixel_format.abi_format()
    ch = 4 if fmt == abi.FORMAT_RGBA_U8 else 3
    dt = {abi.FORMAT_RGB_F32: torch.float32, abi.FORMAT_RGB_U16: torch.uint16, abi.FORMAT_RGB_F16: torch.float16}.get(fmt, torch.uint8)
    frames = [ModularParsedFrame(f) for f in files]
    batch = ModularBatch(ctx, lanes_per_warp)
    outs = []
    try:
        for fr in frames:
            if to_host:
                t = torch.empty((fr.height, fr.width, ch), dtype=dt).pin_memory()
            else:
                t = torch.empty((fr.height, fr.width, ch), dtype=dt, device=f"cuda:{ctx.device}")
            outs.append(t)
            batch.add(fr, t.data_ptr(), fr.width * ch * t.element_size(), not to_host,
                      fmt=None if fmt == abi.FORMAT_RGB_U8 else fmt)
        batch.run()
        batch.wait()
    finally:
        batch.close()
    return outs


def decode_thumbnails(ctx: JxgContext, files, pixel_format: JxlPixelFormat = JxlPixelFormat(), to_host: bool = True):
    """1:8 thumbnails of VarDCT .jxl files (the LF image through the output stage, see jxg_modular_batch_add_lf):
    H x W x C torch tensors, H = ceil(height / 8), W = ceil(width / 8) of the display-oriented image. Only the headers,
    LfGlobal and the LF-group sections are parsed; the LF streams are decoded on the GPU."""
    import torch
    fmt = pixel_format.abi_format()
    frames = [LfParsedFrame(f) for f in files]
    ch = 4 if fmt == abi.FORMAT_RGBA_U8 else 3
    dt = {abi.FORMAT_RGB_F32: torch.float32, abi.FORMAT_RGB_U16: torch.uint16, abi.FORMAT_RGB_F16: torch.float16}.get(fmt, torch.uint8)
    batch = ModularBatch(ctx)
    outs = []
    try:
        for fr in frames:
            if to_host:
                t = torch.empty((fr.height, fr.width, ch), dtype=dt).pin_memory()
            else:
                t = torch.empty((fr.height, fr.width, ch), dtype=dt, device=f"cuda:{ctx.device}")
            outs.append(t)
            batch.add_lf(fr, t.data_ptr(), fr.width * ch * t.element_size(), fmt, not to_host)
        batch.run()
        batch.wait()
    finally:
        batch.close()
    return outs


def decode_prefixes(ctx: JxgContext, files, pixel_format: JxlPixelFormat = JxlPixelFormat(), to_host: bool = True,
                    regions=None):
    """Full-resolution pictures of partly received VarDCT files (PrefixParsedFrame: bare codestreams cut anywhere after
    HfGlobal): H x W x C torch tensors of the display-oriented image, decoded in one batch.
    regions: None, or one entry per file: None (the whole image) or (x, y, w, h) in output coordinates, which decodes
    only that rectangle into an h x w x C tensor."""
    import torch
    fmt = pixel_format.abi_format()
    if regions is None:
        regions = [None] * len(files)
    if len(regions) != len(files):
        raise ValueError("regions: one entry per file")
    frames = [PrefixParsedFrame(f) for f in files]
    ch = 4 if fmt == abi.FORMAT_RGBA_U8 else 3
    dt = {abi.FORMAT_RGB_F32: torch.float32, abi.FORMAT_RGB_U16: torch.uint16, abi.FORMAT_RGB_F16: torch.float16}.get(fmt, torch.uint8)
    batch = Batch(ctx, len(frames))
    outs = []
    try:
        for fr, reg in zip(frames, regions):
            h, w = _out_size(fr, reg)
            if to_host:
                t = torch.empty((h, w, ch), dtype=dt).pin_memory()
            else:
                t = torch.empty((h, w, ch), dtype=dt, device=f"cuda:{ctx.device}")
            outs.append(t)
            batch.add(fr, t.data_ptr(), w * ch * t.element_size(), fmt, not to_host, reg)
        batch.run()
        batch.wait()
    finally:
        batch.close()
    return outs
