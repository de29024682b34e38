"""The CUDA VarDCT float path against the float64 restatement in tests/f64_pipeline.py, one stage at a time, each stage fed
the GPU's own input to it:

  A  debug stop after dequant + IDCT: read_xyb(f, 0) against stage A of the GPU's read_coeffs (two runs bit-identical)
  B  FORMAT_XYB_F32_PLANAR (the fused filter kernel) against stage B of the GPU's stage-A planes
  C  FORMAT_RGB_F32 / FORMAT_RGB_U8 against stage C of the GPU's filtered planes

Bound: |got - ref| <= K * 2^-24 * M + 1e-9 with the K of each stage (DESIGN.md section 4); the assertion message reports
the largest err / (2^-24 M). Covers all eight (Gaborish, EPF 0-3) pairs, one-pixel edge tiles of the 64x32 filter tile,
transform profiles 0-3, prefix-coded streams, sRGB / linear / grey / PQ / BT.709 outputs, the fixtures with IDENTITY /
DCT2X2 / AFV varblocks and one batch mixing filter configurations."""
import os

import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import f64_pipeline as fp

pytestmark = pytest.mark.gpu

# (width, height, seed, distance, epf_iters, gab, profile, entropy, colour)
SYNTHETIC = [
    (1, 1, 1, 1.0, 1, 1, 0, 0, 0),
    (3, 3, 2, 1.0, 0, 1, 1, 0, 0),
    (8, 8, 3, 1.0, 2, 0, 0, 0, 0),
    (9, 17, 4, 1.0, 3, 1, 1, 0, 0),
    (63, 65, 5, 1.0, 0, 0, 1, 0, 0),       # Gaborish off, EPF 0
    (263, 131, 6, 1.5, 2, 0, 2, 1, 0),     # Gaborish off, EPF 2; prefix-coded
    (129, 97, 7, 1.0, 1, 0, 1, 0, 0),      # 64k+1 x 32k+1: one-pixel edge tiles of the fused 64x32 filter tile
    (200, 264, 8, 0.7, 3, 0, 3, 0, 1),     # Gaborish off, EPF 3; 128 / 256 families; linear output
    (193, 129, 9, 1.0, 2, 1, 1, 0, 6),     # grey output
    (520, 512, 10, 1.0, 1, 1, 3, 0, 0),    # vector path inside, scalar path on the ragged edges
    (777, 513, 11, 0.5, 0, 1, 2, 0, 0),
    (600, 520, 12, 1.0, 2, 0, 1, 0, 0),    # Gaborish off, EPF 2, several groups
    (160, 96, 13, 1.0, 2, 1, 1, 0, 3),     # P3 + PQ output
    (160, 96, 14, 1.0, 1, 0, 1, 0, 5),     # custom primaries, DCI white, BT.709 output
]
# The fixtures with IDENTITY, DCT2X2 and AFV varblocks. progressive_ac (3.4 MP) also has them but is over the ~2 MP of
# f64 work per case; it is checked against the f64 stages on the oracle (test_f64_pipeline.py), and the GPU against the
# oracle in test_gpu_parity.py.
FIXTURES = ["zoltan_tasi_unsplash", "opsin_inverse", "dice"]


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


def _synthetic(case):
    import synth
    w, h, seed, dist, epf, gab, profile, entropy, colour = case
    return synth.encode_synthetic(w, h, seed, dist, epf, gab, profile, entropy=entropy, colour=colour)


def _run(ctx, frames, fmt, debug_stop=0):
    """One batch over `frames`; returns the batch (still open) and the host outputs."""
    import torch
    import jxl_rs_b200 as j
    b = j.Batch(ctx, len(frames))
    if debug_stop:
        b.set_debug_stop(debug_stop)
    outs = []
    for pf in frames:
        w, h = pf.info.width, pf.info.height
        if fmt == abi.FORMAT_XYB_F32_PLANAR:
            w, h = pf.info.coded_width, pf.info.coded_height
            o = torch.zeros((3, h, w), dtype=torch.float32).pin_memory()
            stride = w * 4
        elif fmt == abi.FORMAT_RGB_F32:
            o = torch.zeros((h, w, 3), dtype=torch.float32).pin_memory()
            stride = w * 12
        else:
            o = torch.zeros((h, w, 3), dtype=torch.uint8).pin_memory()
            stride = w * 3
        b.add(pf, o.data_ptr(), stride, fmt, False)
        outs.append(o)
    b.run()
    b.wait()
    return b, [o.numpy().copy() for o in outs]


def _check_frames(ctx, datas, what):
    """Every frame's output curve must be one stage C restates (sRGB, linear, BT.709, PQ): no case skips stage C."""
    import jxl_rs_b200 as j
    frames = [j.ParsedFrame(d) for d in datas]
    cfgs = {(int(d.gab != 0), min(int(d.epf_iters), 3)) for d in (pf.desc(abi.FORMAT_RGB_F32)[0] for pf in frames)}
    # stage A, twice: the B and C checks below rely on the planes being reproducible
    b, _ = _run(ctx, frames, abi.FORMAT_XYB_F32_PLANAR, debug_stop=2)
    planes = [b.read_xyb(i, 0) for i in range(len(frames))]
    coeffs = [b.read_coeffs(i) for i in range(len(frames))]
    launches_a = b.stats()["kernel_launches"]
    b.rerun_device()
    b.wait()
    for i in range(len(frames)):
        assert np.array_equal(b.read_xyb(i, 0).view(np.uint32), planes[i].view(np.uint32)), f"{what}: stage A not repeatable"
    b.close()
    bx, xyb = _run(ctx, frames, abi.FORMAT_XYB_F32_PLANAR)
    # the fused filter kernel runs once per (Gaborish, EPF) configuration of the batch in each range of frames
    extra = bx.stats()["kernel_launches"] - launches_a
    assert extra % len(cfgs) == 0 and 1 <= extra // len(cfgs) <= len(frames), (what, extra, sorted(cfgs))
    bx.close()
    b32, rgb = _run(ctx, frames, abi.FORMAT_RGB_F32)
    b32.close()
    b8, rgb8 = _run(ctx, frames, abi.FORMAT_RGB_U8)
    b8.close()
    report = []
    for i, pf in enumerate(frames):
        fr = fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0])
        a, ma = fp.stage_a(fr, coeffs[i])
        ra = fp.check("A", planes[i], a, ma, what)
        bb, mb = fp.stage_b(fr, planes[i].astype(np.float64))
        rb = fp.check("B", xyb[i], bb, mb, what)
        c, mc = fp.stage_c(fr, xyb[i].astype(np.float64))
        rc = fp.check("C", rgb[i], c, mc, what)
        fr8 = fp.Frame(pf.desc(abi.FORMAT_RGB_U8)[0])
        c8, mc8 = fp.stage_c(fr8, xyb[i].astype(np.float64))
        fp.check_output(fp.FMT_U8, rgb8[i], c8, mc8, fr8.output_tf, 1, what)
        report.append((ra, rb, rc))
    print(what, "largest err/(2^-24 M) per stage:", report)


@pytest.mark.parametrize("case", SYNTHETIC, ids=[f"{c[0]}x{c[1]}-epf{c[4]}-gab{c[5]}-p{c[6]}-e{c[7]}-c{c[8]}" for c in SYNTHETIC])
def test_synthetic_stages_match_f64(ctx, case):
    _check_frames(ctx, [_synthetic(case)], str(case))


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_stages_match_f64(ctx, name, golden_dir):
    _check_frames(ctx, [open(os.path.join(golden_dir, "jxl", name + ".jxl"), "rb").read()], name)


def test_mixed_filter_batch_matches_f64(ctx):
    """One batch of frames with different (Gaborish, EPF) pairs: the filter kernel runs once per configuration and CTAs of
    other configurations exit at once; every frame must still meet its own reference."""
    cases = [(96, 80, 20 + k, 1.0, epf, gab, 1, 0, 0) for k, (gab, epf) in enumerate([(0, 0), (1, 2), (0, 2), (1, 0), (0, 3), (1, 1)])]
    _check_frames(ctx, [_synthetic(c) for c in cases], "mixed batch")
