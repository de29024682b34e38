"""1:8 thumbnails of VarDCT frames on the GPU (jxg_lf_parse_file + jxg_modular_batch_add_lf): the device LF planes
are bit-identical to the host front end's (jxg_parsed_desc lf[3]); every format, orientation and transfer curve is
within the float64 output stage's bounds; the HF bytes are never read; thumbnails mix with Modular frames and regions
in one batch; a corrupt LF stream is reported by its LF-group index."""
import os

import numpy as np
import pytest

import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from tests import f64_pipeline as fp
from tests.test_lf_thumbnail import (GOLDEN, expected_thumbnail, lf_code, lf_end, lf_entropy_frames, lf_planes, parse,
                                     synthetic_frames)

pytestmark = pytest.mark.gpu

RGB_FORMATS = [abi.FORMAT_RGB_U8, abi.FORMAT_RGBA_U8, abi.FORMAT_RGB_F32, abi.FORMAT_RGB_U16, abi.FORMAT_RGB_F16]
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def ctx():
    c = j.JxgContext(0)
    yield c
    c.close()


def _geometry(fr, fmt):
    """(rows, width in pixels) of a thumbnail buffer."""
    if fmt == abi.FORMAT_XYB_F32_PLANAR:
        return 3 * fr.coded_height, fr.coded_width
    return fr.height, fr.width


def _alloc(fr, fmt, pad, device):
    import torch
    rows, w = _geometry(fr, fmt)
    stride = w * abi.BYTES_PER_PIXEL[fmt] + pad
    t = torch.full((rows, stride), SENTINEL, dtype=torch.uint8)
    return (t.cuda() if device else t.pin_memory()), stride


def _samples(fr, fmt, buf):
    """The thumbnail's samples: (3, h, w) float32 for XYB planar, else (h, w, ch) in the format's dtype."""
    rows, w = _geometry(fr, fmt)
    a = buf.cpu().numpy()[:, :w * abi.BYTES_PER_PIXEL[fmt]].copy()
    if fmt == abi.FORMAT_XYB_F32_PLANAR:
        return a.view(np.float32).reshape(3, fr.coded_height, w)
    dt = {abi.FORMAT_RGB_F32: np.float32, abi.FORMAT_RGB_U16: np.uint16, abi.FORMAT_RGB_F16: np.uint16}.get(fmt, np.uint8)
    return a.view(dt).reshape(rows, w, -1)


def thumbnails(ctx, files, fmt, pad=0, device=False):
    """One Modular batch of the thumbnails of `files`; returns their sample arrays."""
    frames = [j.LfParsedFrame(f) for f in files]
    b = j.ModularBatch(ctx)
    bufs = []
    try:
        for fr in frames:
            buf, stride = _alloc(fr, fmt, pad, device)
            bufs.append(buf)
            b.add_lf(fr, buf.data_ptr(), stride, fmt, device)
        b.run()
        b.wait()
    finally:
        b.close()
    return [_samples(fr, fmt, buf) for fr, buf in zip(frames, bufs)]


def vardct_fixtures():
    out = []
    for p in GOLDEN:
        data = open(p, "rb").read()
        if parse(j.ParsedFrame, data)[1] == 0:
            out.append((os.path.basename(p), data))
    return out


def test_lf_planes_bit_identical(ctx):
    cases = vardct_fixtures() + synthetic_frames()
    assert len(cases) > 20
    got = thumbnails(ctx, [d for _, d in cases], abi.FORMAT_XYB_F32_PLANAR)
    for (name, data), g in zip(cases, got):
        want, _ = lf_planes(data)
        assert g.shape == want.shape, name
        bad = g.view(np.uint32) != want.view(np.uint32)
        assert not bad.any(), f"{name}: {int(bad.sum())} LF samples differ, first at {np.argwhere(bad)[0].tolist()}"


@pytest.mark.parametrize("fmt", RGB_FORMATS)
def test_output_stage(ctx, fmt):
    """All orientations, and the transfer curves of the colour encodings the synthetic writer reaches (sRGB, linear,
    gamma, PQ, HLG, BT.709, grey, DCI)."""
    cases = [synth.encode_synthetic(300, 180, 60 + o, orientation=o) for o in range(1, 9)]
    cases += [synth.encode_synthetic(260, 170, 70 + c, colour=c) for c in range(8)]
    got = thumbnails(ctx, cases, fmt)
    for i, (data, g) in enumerate(zip(cases, got)):
        ref, mag, tf, o = expected_thumbnail(data, fmt)
        fp.check_output(fmt, g, ref, mag, tf, o, what=f"case {i}")


@pytest.mark.parametrize("case", ["ans"] + [name for name, _ in lf_entropy_frames()])
def test_hf_bytes_unused(ctx, case):
    rng = np.random.default_rng(3)
    data = (synth.encode_synthetic(4100, 2200, 80, profile=0) if case == "ans"
            else dict(lf_entropy_frames())[case])
    end = lf_end(data)
    noisy = data[:end] + rng.integers(0, 256, len(data) - end, dtype=np.uint8).tobytes()
    for fmt in (abi.FORMAT_RGB_U8, abi.FORMAT_XYB_F32_PLANAR):
        clean, cut, rnd = thumbnails(ctx, [data, data[:end], noisy], fmt)
        assert clean.tobytes() == cut.tobytes() == rnd.tobytes()


def test_lz77_lf_streams_take_the_lz77_launch(ctx):
    """The LF streams of the LZ77 frames are counted as LZ77 streams of the batch (they go to the LZ77 decode launch,
    each with its own symbol window), the others are not."""
    frames = dict(lf_entropy_frames())
    for name, want in (("lf-e1-t0", False), ("lf-e2-t0", True), ("lf-e3-t1", True)):
        fr = j.LfParsedFrame(frames[name])
        buf, stride = _alloc(fr, abi.FORMAT_RGB_U8, 0, False)
        b = j.ModularBatch(ctx)
        try:
            b.add_lf(fr, buf.data_ptr(), stride, abi.FORMAT_RGB_U8, False)
            st = b.lz77_stats()
        finally:
            b.close()
        n_lf = -(-fr.coded_width // 256) * -(-fr.coded_height // 256)
        assert st["lz77_streams"] == (n_lf if want else 0), name
        assert (st["window_bytes"] > 0) == want, name


@pytest.mark.parametrize("pixel_format", [j.JxlPixelFormat("RGB", "U8"), j.JxlPixelFormat("RGBA", "U8"),
                                          j.JxlPixelFormat("RGB", "U16"), j.JxlPixelFormat("RGB", "F16"),
                                          j.JxlPixelFormat("RGB", "F32")])
def test_decode_thumbnails(ctx, pixel_format):
    """decode_thumbnails gives the tensors of the batch entry point: shape (height, width, channels) of the display
    thumbnail, the format's dtype, the same samples for host and device outputs."""
    import torch
    files = [synth.encode_synthetic(700, 500, 96, orientation=6), synth.encode_synthetic(2100, 300, 97)]
    fmt = pixel_format.abi_format()
    want = thumbnails(ctx, files, fmt)
    for to_host in (True, False):
        got = j.decode_thumbnails(ctx, files, pixel_format=pixel_format, to_host=to_host)
        for f, g, w in zip(files, got, want):
            fr = j.LfParsedFrame(f)
            assert tuple(g.shape) == (fr.height, fr.width, 4 if fmt == abi.FORMAT_RGBA_U8 else 3)
            assert g.is_cuda != to_host
            a = g.cpu()
            a = a.view(torch.uint16) if a.dtype == torch.float16 else a
            assert a.dtype == {abi.FORMAT_RGB_F32: torch.float32, abi.FORMAT_RGB_U16: torch.uint16}.get(
                fmt, torch.uint16 if fmt == abi.FORMAT_RGB_F16 else torch.uint8)
            assert a.numpy().tobytes() == w.tobytes()


def _modular_single(ctx, mfr, region, device, pad):
    import torch
    w, h = (mfr.width, mfr.height) if region is None else region[2:]
    t = torch.full((h, w * 3 + pad), SENTINEL, dtype=torch.uint8)
    t = t.cuda() if device else t.pin_memory()
    return t, w * 3 + pad


def _mixed(ctx, lf_files, mfile, device, pad, fmt):
    """A batch of thumbnails, a whole Modular frame and a Modular region; then each alone. Returns (mixed, alone)."""
    region = (37, 21, 150, 90)
    lfs = [j.LfParsedFrame(f) for f in lf_files]
    mfr = j.ModularParsedFrame(mfile)

    def run(items):
        b = j.ModularBatch(ctx)
        outs = []
        try:
            for kind, arg in items:
                if kind == "lf":
                    buf, stride = _alloc(arg, fmt, pad, device)
                    b.add_lf(arg, buf.data_ptr(), stride, fmt, device)
                else:
                    buf, stride = _modular_single(ctx, mfr, arg, device, pad)
                    b.add(mfr, buf.data_ptr(), stride, device, arg)
                outs.append(buf)
            b.run()
            b.wait()
        finally:
            b.close()
        return [o.cpu().numpy().tobytes() for o in outs]

    items = [("lf", lfs[0]), ("modular", None), ("lf", lfs[1]), ("modular", region), ("lf", lfs[2])]
    return run(items), [run([it])[0] for it in items]


@pytest.mark.parametrize("device,pad", [(False, 0), (True, 0), (False, 12), (True, 4)])
def test_mixed_batches(ctx, device, pad):
    lf_files = [synth.encode_synthetic(2100, 300, 90), synth.encode_synthetic(700, 500, 91, orientation=6),
                synth.encode_synthetic(4100, 2200, 92, profile=0)]
    mfile = synth.encode_modular(600, 520, 7, 6, 1, 2)
    for fmt in (abi.FORMAT_RGB_F16, abi.FORMAT_RGB_U8):
        mixed, alone = _mixed(ctx, lf_files, mfile, device, pad, fmt)
        assert mixed == alone
    try:
        ctx.set_sm_budget(1)
        for fill in (0x00, 0xFF):
            ctx.set_pool_fill(fill)
            assert _mixed(ctx, lf_files, mfile, device, pad, abi.FORMAT_RGB_U8) == (mixed, alone)
    finally:
        ctx.set_pool_fill(-1)
        ctx.set_sm_budget(0)


def test_bad_output_refused_and_batch_unchanged(ctx):
    import torch
    data = synth.encode_synthetic(700, 500, 93)
    fr = j.LfParsedFrame(data)
    good = thumbnails(ctx, [data], abi.FORMAT_RGB_F32)[0]
    b = j.ModularBatch(ctx)
    try:
        buf = torch.zeros((fr.height, fr.width * 12 + 8), dtype=torch.uint8).pin_memory()
        for stride in (fr.width * 12 - 4, fr.width * 12 + 2):  # too small; not a multiple of the sample size
            with pytest.raises(abi.JxgError) as e:
                b.add_lf(fr, buf.data_ptr(), stride, abi.FORMAT_RGB_F32, False)
            assert e.value.code == -9  # JXG_ERR_INVALID_OUTPUT
        dev = torch.zeros(fr.height * fr.width * 12 + 64, dtype=torch.uint8, device="cuda")
        with pytest.raises(abi.JxgError) as e:
            b.add_lf(fr, dev.data_ptr() + 2, fr.width * 12, abi.FORMAT_RGB_F32, True)
        assert e.value.code == -9
        b.add_lf(fr, buf.data_ptr(), fr.width * 12 + 8, abi.FORMAT_RGB_F32, False)
        b.run()
        b.wait()
        with pytest.raises(abi.JxgError) as e:
            b.read_planes(0)
        assert e.value.code == -22  # JXG_ERR_ARGUMENT
    finally:
        b.close()
    got = buf.numpy()[:, :fr.width * 12].copy().view(np.float32).reshape(fr.height, fr.width, 3)
    assert got.tobytes() == good.tobytes()


def _randomised(data, a, b, seed):
    return data[:a] + np.random.default_rng(seed).integers(0, 256, b - a, dtype=np.uint8).tobytes() + data[b:]


@pytest.mark.parametrize("w,h,k", [(600, 400, 0), (4100, 2200, 5)])
def test_corrupt_lf_group(ctx, w, h, k):
    """The last LF-group section (group k) replaced by random bytes behind its stream header (the longest tail whose
    randomisation the host parse still accepts, less 16 bytes): its LF stream fails on the device, wait names LF group
    k, and the other thumbnail of the batch is still right."""
    data = synth.encode_synthetic(w, h, 94, profile=0)
    other = synth.encode_synthetic(700, 500, 95)
    want = thumbnails(ctx, [other], abi.FORMAT_RGB_U8)[0]
    end = lf_end(data)
    lo, hi = 1, end  # largest tail length that still parses
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if lf_code(_randomised(data, end - mid, end, k)) == 0:
            lo = mid
        else:
            hi = mid - 1
    assert lo > 64
    bad = _randomised(data, end - lo + 16, end, k)
    frames = [j.LfParsedFrame(other), j.LfParsedFrame(bad)]
    b = j.ModularBatch(ctx)
    bufs = []
    try:
        for fr in frames:
            buf, stride = _alloc(fr, abi.FORMAT_RGB_U8, 0, False)
            bufs.append(buf)
            b.add_lf(fr, buf.data_ptr(), stride, abi.FORMAT_RGB_U8, False)
        b.run()
        with pytest.raises(abi.JxgError):
            b.wait()
        assert b.last_failure == (1, k)
    finally:
        b.close()
    assert _samples(frames[0], abi.FORMAT_RGB_U8, bufs[0]).tobytes() == want.tobytes()
