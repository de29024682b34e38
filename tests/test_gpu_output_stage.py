"""The CUDA output stage against stage C of tests/f64_pipeline.py, fed the GPU's own filtered planes: every output curve
(linear, sRGB, gamma 1/2.2 and DCI 1/2.6, BT.709, PQ, HLG at 1000 nits (e < 0) and at 100 nits (e > 0)) in every format
(U8, RGBA_U8, F32, U16, F16, XYB planar), through both store paths of the fused filter kernel; orientations 1-8; frames
whose LF is overwritten with edge values (black, negatives, out of gamut, above 1, f16 subnormals, both sides of every
curve's breakpoint); and the rejection of output rows the device cannot store to.

Store paths (kernels.cu locate_tile): the vector path takes interior 64x32 tiles of Gaborish + EPF 2 frames whose output
row is 16-byte aligned (4-byte for RGB_U8) in U8 / RGBA / F32 / XYB. The same frame with a row stride padded by 4 bytes
(1 byte for RGB_U8) takes the scalar path everywhere; U16 / F16 always do."""
import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import f64_pipeline as fp
from tests.test_gpu_f64_stages import ctx  # noqa: F401  (the module-scoped context fixture)

pytestmark = pytest.mark.gpu

FORMATS = [abi.FORMAT_RGB_U8, abi.FORMAT_RGBA_U8, abi.FORMAT_RGB_F32, abi.FORMAT_RGB_U16, abi.FORMAT_RGB_F16,
           abi.FORMAT_XYB_F32_PLANAR]
# (name, output_tf, output_gamma, intensity_target)
CURVES = [("linear", fp.TF_LINEAR, 1.0, 255.0), ("srgb", fp.TF_SRGB, 1.0, 255.0), ("gamma2.2", fp.TF_GAMMA, 1 / 2.2, 255.0),
          ("dci", fp.TF_GAMMA, 1 / 2.6, 255.0), ("bt709", fp.TF_BT709, 1.0, 255.0), ("pq", fp.TF_PQ, 1.0, 1000.0),
          ("hlg1000", fp.TF_HLG, 1.0, 1000.0), ("hlg100", fp.TF_HLG, 1.0, 100.0)]
KTW, KTH = 64, 32  # fused filter tile (launch.h kFusedTileW / kFusedTileH)
SENTINEL = 0xA5
JXG_ERR_INVALID_OUTPUT = -9  # include/jxg.h


def vector_tiles(w, h, gab, epf, fmt, stride, ptr_align=256):
    """kernels.cu locate_tile: number of tiles that take the vector path. ptr_align: alignment of the output base (host
    outputs are staged in a 256-byte aligned device buffer)."""
    if not (gab and min(epf, 3) == 2) or fmt not in (abi.FORMAT_RGB_U8, abi.FORMAT_RGBA_U8, abi.FORMAT_RGB_F32,
                                                       abi.FORMAT_XYB_F32_PLANAR):
        return 0
    need = 4 if fmt == abi.FORMAT_RGB_U8 else 16
    if stride % need or ptr_align % need:
        return 0
    halo = 4  # Gaborish 1 + EPF1 2 + EPF2 1
    xs = [x for x in range(0, w, KTW) if x - halo >= 0 and x + KTW + halo <= w]
    ys = [y for y in range(0, h, KTH) if y - halo >= 0 and y + KTH + halo <= h]
    return len(xs) * len(ys)


def _alloc(fmt, w, h, stride, device):
    """A byte buffer of h rows (3h for XYB planar) of `stride` bytes, filled with SENTINEL."""
    import torch
    rows = 3 * h if fmt == abi.FORMAT_XYB_F32_PLANAR else h
    if device:
        return torch.full((rows, stride), SENTINEL, dtype=torch.uint8, device="cuda")
    return torch.full((rows, stride), SENTINEL, dtype=torch.uint8).pin_memory()


def _view(fmt, buf, w, h):
    """The samples of a filled buffer: (h, w, ch) in the format's dtype, or (3, h, w) float32 for XYB planar."""
    bpp = abi.BYTES_PER_PIXEL[fmt]
    a = buf[:, :w * bpp].copy()
    if fmt == abi.FORMAT_XYB_F32_PLANAR:
        return a.view(np.float32).reshape(3, h, w)
    dt = {abi.FORMAT_RGB_F32: np.float32, abi.FORMAT_RGB_U16: np.uint16, abi.FORMAT_RGB_F16: np.uint16}.get(fmt, np.uint8)
    return a.view(dt).reshape(h, w, 4 if fmt == abi.FORMAT_RGBA_U8 else 3)


def decode(ctx, pf, fmt, edits=None, lf=None, pad=0, device=False, debug_stop=0):  # noqa: F811 (ctx: the fixture's value)
    """One frame through Batch.add_desc with fields of its descriptor overwritten. Returns (samples, batch, desc);
    checks that the row padding (device outputs) kept its sentinel. The batch is left open for read_xyb / read_coeffs."""
    import jxl_rs_b200 as j
    d, hf, off, ln, n = pf.desc(fmt)
    fp.edit_desc(d, lf, **(edits or {}))
    cw, ch = int(d.width), int(d.height)
    o = int(d.orientation) if fmt != abi.FORMAT_XYB_F32_PLANAR else 1
    w, h = (ch, cw) if o >= 5 else (cw, ch)
    stride = w * abi.BYTES_PER_PIXEL[fmt] + pad
    buf = _alloc(fmt, w, h, stride, device)
    b = j.Batch(ctx, 1)
    if debug_stop:
        b.set_debug_stop(debug_stop)
    b.add_desc(d, hf, off, ln, n, buf.data_ptr(), stride, device)
    b.frames.append(pf)
    b.run()
    b.wait()
    host = buf.cpu().numpy()
    if device and pad:
        assert (host[:, w * abi.BYTES_PER_PIXEL[fmt]:] == SENTINEL).all(), f"format {fmt}: row padding overwritten"
    return _view(fmt, host, w, h), b, d


def _frame(w, h, seed, dist, epf, gab, profile=1):
    import jxl_rs_b200 as j
    import synth
    return j.ParsedFrame(synth.encode_synthetic(w, h, seed, dist, epf, gab, profile))


def _curve_edits(curve):
    _, tf, g, it = curve
    return {"output_tf": tf, "output_gamma": g, "intensity_target": it, "output_luminances": fp.BT2100_LUMINANCES}


def _check_curve_matrix(ctx, pf, gab, epf, curve, lf=None, regions=False):
    """All formats of one curve on one frame, through the vector path (tight rows) and the scalar path (padded rows).
    Each output is checked against stage C (stage B for XYB) of the filtered planes of the same path."""
    name = curve[0]
    edits = _curve_edits(curve)
    planes, b, d = decode(ctx, pf, abi.FORMAT_XYB_F32_PLANAR, edits, lf, debug_stop=2)
    planes = b.read_xyb(0, 0)
    fr = fp.Frame(d)
    if lf is not None:  # the edited frame through stage A too
        a, ma = fp.stage_a(fr, b.read_coeffs(0))
        fp.check("A", planes, a, ma, f"{name} edge frame")
    b.close()
    bb, mb = fp.stage_b(fr, planes.astype(np.float64))
    w, h = fr.width, fr.height
    ratios, counts = {}, None
    for pad_kind in ("tight", "padded"):
        refs = {}
        for fmt in FORMATS:
            pad = 0 if pad_kind == "tight" else (1 if fmt == abi.FORMAT_RGB_U8 else 4)
            nvec = vector_tiles(w, h, gab, epf, fmt, w * abi.BYTES_PER_PIXEL[fmt] + pad)
            if pad_kind == "tight" and fmt != abi.FORMAT_RGB_U16 and fmt != abi.FORMAT_RGB_F16 and gab and epf == 2:
                assert nvec > 0, f"{name}: the vector case has no vector tiles"
            got, b, dfmt = decode(ctx, pf, fmt, edits, lf, pad=pad, device=pad_kind == "padded")
            b.close()
            what = f"{name} {pad_kind} format {fmt}"
            if fmt == abi.FORMAT_XYB_F32_PLANAR:
                fp.check("B", got, bb, mb, what)
                refs["xyb"] = got
                continue
            frf = fp.Frame(dfmt)
            key = (frf.output_tf, frf.output_gamma, frf.intensity_target)
            if key not in refs:
                xyb = refs.get("xyb")
                if xyb is None:
                    xyb, bx, _ = decode(ctx, pf, abi.FORMAT_XYB_F32_PLANAR, edits, lf, pad=0 if pad_kind == "tight" else 4)
                    bx.close()
                    refs["xyb"] = xyb
                refs[key] = fp.stage_c(frf, xyb.astype(np.float64), full=True) + (xyb,)
            c, mc, _, amb, xyb = refs[key]
            r = fp.check_output(fmt, got, c, mc, frf.output_tf, 1, what)
            if fmt == abi.FORMAT_RGB_F32:
                ratios[pad_kind] = r
                if regions:
                    counts = fp.edge_regions(fp.linear_rgb_f64(frf, xyb.astype(np.float64)), c, frf.output_tf,
                                             fp.BT2100_LUMINANCES)
            if fmt == abi.FORMAT_RGBA_U8:
                refs["rgba"] = got
            if fmt == abi.FORMAT_RGB_U8:
                refs["u8"] = got
        assert np.array_equal(refs["rgba"][..., :3], refs["u8"]) and (refs["rgba"][..., 3] == 255).all(), \
            f"{name} {pad_kind}: RGBA is not RGB_U8 plus alpha 255"
    print(name, "largest err/(2^-24 M) of the f32 output:", ratios, counts or "")
    return ratios, counts


MATRIX_FRAMES = [(320, 192, 50, 1.0, 2, 1), (257, 131, 51, 1.0, 1, 0)]  # vector + scalar paths; scalar only


@pytest.mark.parametrize("frame", MATRIX_FRAMES, ids=[f"{f[0]}x{f[1]}-gab{f[5]}-epf{f[4]}" for f in MATRIX_FRAMES])
@pytest.mark.parametrize("curve", CURVES, ids=[c[0] for c in CURVES])
def test_output_matrix_matches_f64(ctx, frame, curve):
    w, h, seed, dist, epf, gab = frame
    _check_curve_matrix(ctx, _frame(w, h, seed, dist, epf, gab), gab, epf, curve)


@pytest.mark.parametrize("curve", CURVES, ids=[c[0] for c in CURVES])
def test_edge_value_frames_match_f64(ctx, curve):
    """A 256x128 Gaborish + EPF 2 frame (DCT8 only, distance 4) whose LF field is overwritten with the edge targets of
    f64_pipeline.edge_targets for the curve's intensity target. Every edge region must hold samples, so the frame cannot
    silently lose its edge coverage (f16 subnormals: not for the curves of f64_pipeline.NO_F16_SUBNORMALS)."""
    pf = _frame(256, 128, 5, 4.0, 2, 1, profile=0)
    fr = fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0])
    lf = fp.edge_lf(fr, fp.edge_targets(), curve[3])
    _, counts = _check_curve_matrix(ctx, pf, 1, 2, curve, lf=lf, regions=True)
    empty = [k for k, v in counts.items() if v == 0 and not (k == "f16_subnormal" and curve[0] in fp.NO_F16_SUBNORMALS)]
    assert not empty, f"{curve[0]}: empty edge regions {empty}"


def test_orientations_are_exact_permutations(ctx):
    """Orientations 1-8, every format, host and device outputs, rows padded by 16 or 32 bytes (sentinel untouched on the
    device; a host output's padding receives the device staging rows): each output is bit-identical to orient(output at
    orientation 1). XYB planar ignores the orientation. 320x192 Gaborish + EPF 2 with 16-byte multiples of padding: the
    staged coded image and the orientation-1 output take the same (vector) store path."""
    pf = _frame(320, 192, 52, 1.0, 2, 1)
    for fmt in FORMATS:
        base, b, _ = decode(ctx, pf, fmt, {"orientation": 1})
        b.close()
        for o in range(1, 9):
            for device in (False, True):
                got, b, _ = decode(ctx, pf, fmt, {"orientation": o}, pad=16 * (1 + o % 2), device=device)
                b.close()
                want = base if fmt == abi.FORMAT_XYB_F32_PLANAR else fp.orient(base, o)
                assert got.shape == want.shape and np.array_equal(got.view(np.uint8), np.ascontiguousarray(want).view(np.uint8)), \
                    f"format {fmt} orientation {o} device {device}"


def test_sixteen_bit_orientations_match_f64(ctx):
    """U16 and F16 at every orientation against stage C (interval rule), so the 6-byte orientation pass is held to
    the f64 reference and not only to the orientation-1 output."""
    pf = _frame(200, 120, 53, 1.0, 2, 1)
    xyb, b, _ = decode(ctx, pf, abi.FORMAT_XYB_F32_PLANAR)
    b.close()
    for fmt in (abi.FORMAT_RGB_U16, abi.FORMAT_RGB_F16):
        for o in range(1, 9):
            got, b, d = decode(ctx, pf, fmt, {"orientation": o})
            b.close()
            fr = fp.Frame(d)
            c, mc = fp.stage_c(fr, xyb.astype(np.float64))
            fp.check_output(fmt, got, c, mc, fr.output_tf, o, f"format {fmt} orientation {o}")


@pytest.mark.parametrize("fmt,bad_stride,bad_ptr", [
    (abi.FORMAT_RGBA_U8, 2, 2), (abi.FORMAT_RGB_F32, 2, 1), (abi.FORMAT_XYB_F32_PLANAR, 1, 2),
    (abi.FORMAT_RGB_U16, 1, 1), (abi.FORMAT_RGB_F16, 1, 1)])
def test_misaligned_outputs_are_rejected(ctx, fmt, bad_stride, bad_ptr):
    """A row stride that is not a multiple of the sample size, or a device pointer not aligned to it, is refused by
    add with JXG_ERR_INVALID_OUTPUT. Nothing is run: the batch is closed right after the refused add."""
    import torch
    import jxl_rs_b200 as j
    pf = _frame(96, 80, 54, 1.0, 2, 1)
    bpp = abi.BYTES_PER_PIXEL[fmt]
    rows = 3 * 80 if fmt == abi.FORMAT_XYB_F32_PLANAR else 80
    buf = torch.zeros(rows * (96 * bpp + 16) + 16, dtype=torch.uint8, device="cuda")
    for ptr, stride, device in ((buf.data_ptr(), 96 * bpp + bad_stride, True),
                                (buf.data_ptr(), 96 * bpp + bad_stride, False),
                                (buf.data_ptr() + bad_ptr, 96 * bpp, True)):
        b = j.Batch(ctx, 1)
        with pytest.raises(abi.JxgError) as e:
            if device:
                b.add(pf, ptr, stride, fmt, True)
            else:
                host = torch.zeros(rows * stride, dtype=torch.uint8).pin_memory()
                b.add(pf, host.data_ptr(), stride, fmt, False)
        b.close()
        assert e.value.code == JXG_ERR_INVALID_OUTPUT, str(e.value)
    # aligned strides with padding and odd RGB_U8 strides stay accepted (and are decoded in the matrix tests)
    b = j.Batch(ctx, 1)
    b.add(pf, buf.data_ptr(), 96 * bpp + 4, fmt, True)
    b.close()
