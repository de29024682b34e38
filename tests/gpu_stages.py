"""Stage-by-stage check of the CUDA VarDCT float path against the float64 restatement in tests/f64_pipeline.py (not a
test module; used by test_gpu_f64_stages.py and test_gpu_dequant_matrices.py). Each stage is fed the GPU's own input:

  A  debug stop after dequant + IDCT: read_xyb(f, 0) against stage A of the GPU's read_coeffs (two runs bit-identical)
  B  FORMAT_XYB_F32_PLANAR (the fused filter kernel) against stage B of the GPU's stage-A planes
  C  FORMAT_RGB_F32 / FORMAT_RGB_U8 against stage C of the GPU's filtered planes

Bound: |got - ref| <= K * 2^-24 * M + 1e-9 with the K of each stage (DESIGN.md section 4); the assertion message reports
the largest err / (2^-24 M)."""
import numpy as np

from jxl_rs_b200 import abi
from tests import f64_pipeline as fp


def run(ctx, frames, fmt, debug_stop=0):
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


def check_frames(ctx, datas, what, encodings=None):
    """Every frame's output curve must be one stage C restates (sRGB, linear, BT.709, PQ): no case skips stage C.
    encodings: per frame, the 17 dequantisation encodings it was written with (None: all library tables); stage A is
    built from them. The GPU's coefficients must equal the oracle's. Returns the largest ratio per frame and stage."""
    import jxl_rs_b200 as j
    from tests import oracle_binding as ob
    encodings = encodings or [None] * len(datas)
    frames = [j.ParsedFrame(d) for d in datas]
    cfgs = {(int(d.gab != 0), min(int(d.epf_iters), 3)) for d in (pf.desc(abi.FORMAT_RGB_F32)[0] for pf in frames)}
    # stage A, twice: the B and C checks below rely on the planes being reproducible
    b, _ = run(ctx, frames, abi.FORMAT_XYB_F32_PLANAR, debug_stop=2)
    planes = [b.read_xyb(i, 0) for i in range(len(frames))]
    coeffs = [b.read_coeffs(i) for i in range(len(frames))]
    launches_a = b.stats()["kernel_launches"]
    b.rerun_device()
    b.wait()
    for i in range(len(frames)):
        assert np.array_equal(b.read_xyb(i, 0).view(np.uint32), planes[i].view(np.uint32)), f"{what}: stage A not repeatable"
    b.close()
    for i, data in enumerate(datas):
        _, taps = ob.decode_file(data, abi.FORMAT_RGB_F32, taps=True)
        assert np.array_equal(coeffs[i], taps["coeffs"]), f"{what}: frame {i} coefficients differ from the oracle"
    bx, xyb = run(ctx, frames, abi.FORMAT_XYB_F32_PLANAR)
    # the fused filter kernel runs once per (Gaborish, EPF) configuration of the batch in each range of frames
    extra = bx.stats()["kernel_launches"] - launches_a
    assert extra % len(cfgs) == 0 and 1 <= extra // len(cfgs) <= len(frames), (what, extra, sorted(cfgs))
    bx.close()
    b32, rgb = run(ctx, frames, abi.FORMAT_RGB_F32)
    b32.close()
    b8, rgb8 = run(ctx, frames, abi.FORMAT_RGB_U8)
    b8.close()
    report = []
    for i, pf in enumerate(frames):
        fr = fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0], encodings=encodings[i])
        a, ma = fp.stage_a(fr, coeffs[i])
        ra = fp.check("A", planes[i], a, ma, what)
        bb, mb = fp.stage_b(fr, planes[i].astype(np.float64))
        rb = fp.check("B", xyb[i], bb, mb, what)
        c, mc = fp.stage_c(fr, xyb[i].astype(np.float64))
        rc = fp.check("C", rgb[i], c, mc, what)
        fr8 = fp.Frame(pf.desc(abi.FORMAT_RGB_U8)[0], encodings=encodings[i])
        c8, mc8 = fp.stage_c(fr8, xyb[i].astype(np.float64))
        fp.check_output(fp.FMT_U8, rgb8[i], c8, mc8, fr8.output_tf, 1, what)
        report.append((round(ra, 2), round(rb, 2), round(rc, 2)))
    print(what, "largest err/(2^-24 M) per stage (A, B, C):", report)
    return report
