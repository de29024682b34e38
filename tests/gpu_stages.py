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
    """One batch over `frames` (parsed frames, or (frame, region) pairs); returns the batch (still open) and the host
    outputs."""
    import torch
    import jxl_rs_b200 as j
    b = j.Batch(ctx, len(frames))
    if debug_stop:
        b.set_debug_stop(debug_stop)
    outs = []
    for item in frames:
        pf, reg = item if isinstance(item, tuple) else (item, None)
        w, h = (pf.info.width, pf.info.height) if reg is None else reg[2:]
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
        b.add(pf, o.data_ptr(), stride, fmt, False, reg)
        outs.append(o)
    b.run()
    b.wait()
    return b, [o.numpy().copy() for o in outs]


def check_frames(ctx, datas, what, encodings=None, headers=None, cuts=None, lf_images=None, weights8=None,
                 regions=None):
    """Every frame's output curve must be one stage C restates (sRGB, linear, BT.709, PQ): no case skips stage C.
    encodings: per frame, the 17 dequantisation encodings it was written with (None: all library tables); stage A is
    built from them. headers: per frame, the header fields it was written with (f64_pipeline.Frame's header), None for
    defaults. The GPU's coefficients must equal the oracle's. Returns the largest ratio per frame and stage.
    Prefix frames (tests/f64_prefix.py): cuts, per frame None (the whole file) or the length of the prefix decoded
    through jxg_parse_file_prefix. Stage A is then f64_prefix.stage_a with the prefix's pass counts (weights8: per frame
    its upsampling weights, None for the defaults), and the coefficients of each group with k passes must equal the
    oracle's fed the first k passes. lf_images: per frame None or the (planes, magnitude) of a float64 LF image
    (f64_prefix.token_lf_image) that replaces the descriptor's in stage A. regions: per frame, regions (display
    coordinates) decoded to RGB_U8 in one more batch, each within the bounds of the crop of the frame's stage C."""
    import jxl_rs_b200 as j
    from tests import f64_prefix as fpx
    from tests import oracle_binding as ob
    n = len(datas)
    encodings = encodings or [None] * n
    headers = headers or [None] * n
    cuts = cuts or [None] * n
    lf_images = lf_images or [None] * n
    weights8 = weights8 or [None] * n
    regions = regions or [[]] * n
    wholes = [j.ParsedFrame(d) for d in datas]  # the descriptor: a prefix holds every section it is made from
    frames = [pf if cut is None else j.PrefixParsedFrame(d[:cut]) for pf, d, cut in zip(wholes, datas, cuts)]
    cfgs = {(int(d.gab != 0), min(int(d.epf_iters), 3)) for d in (pf.desc(abi.FORMAT_RGB_F32)[0] for pf in wholes)}
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
        if cuts[i] is not None:
            from tests.test_gpu_prefix import oracle_passes
            k = frames[i].passes
            assert not coeffs[i][k == 0].any(), f"{what}: frame {i} has coefficients in a group without a pass"
            for kk in sorted(set(k.tolist()) - {0}):
                want = oracle_passes(data, kk)["coeffs"]
                assert np.array_equal(coeffs[i][k == kk], want[k == kk]), f"{what}: frame {i} {kk}-pass coefficients"
            continue
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
    regs = [(i, r) for i in range(n) for r in regions[i]]
    if regs:
        br, rgb8_regions = run(ctx, [(frames[i], r) for i, r in regs], abi.FORMAT_RGB_U8)
        br.close()
    for i, pf in enumerate(wholes):
        fr = fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0], encodings=encodings[i], header=headers[i])
        if lf_images[i] is not None:
            fpx.use_lf_image(fr, *lf_images[i][:2])
        if cuts[i] is None:
            a, ma = fp.stage_a(fr, coeffs[i])
        else:
            a, ma = fpx.stage_a(fr, coeffs[i], frames[i].passes, weights8[i])
        ra = fp.check("A", planes[i], a, ma, what)
        bb, mb = fp.stage_b(fr, planes[i].astype(np.float64))
        rb = fp.check("B", xyb[i], bb, mb, what)
        c, mc = fp.stage_c(fr, xyb[i].astype(np.float64))
        # samples beyond the f32 range of the sRGB curve (planes of 1e6 and more only): under 1%, left out
        over = fp.srgb_f32_overflow(fr, xyb[i])
        assert over.sum() <= over.size // 100, f"{what}: {int(over.sum())} samples beyond the f32 range of the curve"
        rc = fp.check("C", rgb[i][~over], c[~over], mc[~over], what)
        fr8 = fp.Frame(pf.desc(abi.FORMAT_RGB_U8)[0], encodings=encodings[i], header=headers[i])
        c8, mc8 = fp.stage_c(fr8, xyb[i].astype(np.float64))
        mc8 = np.where(fp.srgb_f32_overflow(fr8, xyb[i]), np.inf, mc8)
        fp.check_output(fp.FMT_U8, rgb8[i], c8, mc8, fr8.output_tf, 1, what)
        for (fi, (x, y, w, h)), got in zip(regs, rgb8_regions if regs else []):
            if fi == i:  # pasted into the whole output (which passed), so that the store's dither sees frame positions
                pasted = rgb8[i].copy()
                pasted[y:y + h, x:x + w] = got
                fp.check_output(fp.FMT_U8, pasted, c8, mc8, fr8.output_tf, fr8.orientation, f"{what} region {(x, y, w, h)}")
        report.append((round(ra, 2), round(rb, 2), round(rc, 2)))
    print(what, "largest err/(2^-24 M) per stage (A, B, C):", report)
    return report
