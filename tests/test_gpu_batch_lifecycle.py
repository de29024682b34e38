"""The lifecycle both batch engines share (BatchCore, csrc/cuda/batch_common.h): a run and reruns on a caller's CUDA
stream read back through the taps as a run on the context's own stream does, since the taps wait for the batch's own
last run; the Modular tables travel in the one pinned blob copy; one live batch per context, across the two engines."""
import numpy as np
import pytest

from jxl_rs_b200 import abi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


def _modular_file(lz77):
    import synth
    return synth.encode_modular(600, 520, 7, rct=6, squeeze=1, tree_kind=2, lz77=lz77)


def _modular_on(ctx, files, stream_ptr, reruns):
    """(i32 planes, u8 device outputs copied to the host, stats) of one ModularBatch run (and `reruns` reruns) on
    `stream_ptr`; the outputs live on the device, so every rerun rewrites them."""
    import torch
    import jxl_rs_b200 as j
    frames = [j.ModularParsedFrame(f) for f in files]
    outs = [torch.zeros((fr.height, fr.width, 3), dtype=torch.uint8, device="cuda:0") for fr in frames]
    torch.cuda.synchronize()
    b = j.ModularBatch(ctx, 2)
    try:
        for fr, o in zip(frames, outs):
            b.add(fr, o.data_ptr(), fr.width * 3, True)
        b.run(stream_ptr)
        for _ in range(reruns):
            b.rerun_device(stream_ptr)
        b.wait()
        planes = [b.read_planes(i) for i in range(len(frames))]
        stats = b.stats()
    finally:
        b.close()
    return planes, [o.cpu().numpy() for o in outs], stats


def test_modular_run_and_reruns_on_a_caller_stream(ctx):
    import torch
    files = [_modular_file(0), _modular_file(1)]
    ref_planes, ref_outs, _ = _modular_on(ctx, files, 0, 0)
    s = torch.cuda.Stream()
    planes, outs, _ = _modular_on(ctx, files, s.cuda_stream, 2)
    for p, rp, o, ro in zip(planes, ref_planes, outs, ref_outs):
        assert np.array_equal(p, rp)
        assert np.array_equal(o, ro)


def test_vardct_read_xyb_after_runs_on_a_caller_stream(ctx):
    import torch
    import synth
    import jxl_rs_b200 as j
    files = [synth.encode_synthetic(256, 256, 1000, 0.5, 2, 1, 1), synth.encode_synthetic(512, 384, 1001, 0.5, 3, 1, 2)]
    frames = [j.ParsedFrame(f) for f in files]

    def xyb(stream_ptr, reruns):
        outs = [torch.empty((fr.height, fr.width, 3), dtype=torch.uint8).pin_memory() for fr in frames]
        b = j.Batch(ctx, len(frames))
        try:
            b.set_debug_stop(2)
            for fr, o in zip(frames, outs):
                b.add(fr, o.data_ptr(), fr.width * 3, abi.FORMAT_RGB_U8, False)
            b.run(stream_ptr)
            for _ in range(reruns):
                b.rerun_device(stream_ptr)
            b.wait()
            return [b.read_xyb(i, 0) for i in range(len(frames))]
        finally:
            b.close()

    ref = xyb(0, 0)
    s = torch.cuda.Stream()
    for got, want in zip(xyb(s.cuda_stream, 2), ref):
        assert np.array_equal(got, want)


@pytest.mark.parametrize("lz77,launches", [((0,), 49), ((1,), 49), ((0, 1), 50)], ids=["plain", "lz77", "mixed"])
def test_modular_uploads_and_launches(ctx, lz77, launches):
    """The blob copy is the whole upload: it holds every section, and it is the same for the same frames. Launches:
    the group-stream decode, then one per level of the inverse plan (RCT and the Squeeze steps) and the store; a batch
    with streams both with and without LZ77 takes one more decode launch."""
    import jxl_rs_b200 as j
    files = [_modular_file(lz) for lz in lz77]
    section_bytes = sum(j.ModularParsedFrame(f).info.hf_bytes for f in files)
    _, _, st_a = _modular_on(ctx, files, 0, 0)
    _, _, st_b = _modular_on(ctx, files, 0, 0)
    assert st_a["h2d_bytes"] == st_b["h2d_bytes"] >= section_bytes
    assert st_a["kernel_launches"] == st_b["kernel_launches"] == launches


def test_one_live_batch_per_context_across_engines(ctx):
    import jxl_rs_b200 as j
    m = j.ModularBatch(ctx)
    try:
        with pytest.raises(abi.JxgError):
            j.Batch(ctx)
    finally:
        m.close()
    b = j.Batch(ctx)
    try:
        with pytest.raises(abi.JxgError):
            j.ModularBatch(ctx)
    finally:
        b.close()
    j.ModularBatch(ctx).close()
    j.Batch(ctx).close()
