"""The oracle's VarDCT float path against the float64 restatement in tests/f64_pipeline.py, one stage at a time, with the
bound |got - ref| <= K * 2^-24 * M + 1e-9 (M: the stage computed on magnitudes; K per stage, DESIGN.md section 4).
Each stage is fed the oracle's own input to that stage (its coefficient, xyb_idct and xyb_filtered taps), so a
failure names the stage. The sensitivity tests plant one fault on the f64 side and check that the bound catches it.
No GPU."""
import ctypes as C

import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import f64_pipeline as fp

GOLDEN = "tests/golden/jxl/"
FIXTURES = ["zoltan_tasi_unsplash", "progressive_ac", "opsin_inverse", "dice", "has_permutation", "grayscale",
            "green_queen_vardct_e3", "3x3_srgb_lossy", "3x3a_srgb_lossy"]
# (width, height, seed, distance, epf_iters, gab, profile, entropy, colour): every (Gaborish, EPF) pair, odd sizes,
# profiles 0-3, the eight colour encodings of the synthetic writer
SYNTHETIC = [(1, 1, 1, 1.0, 1, 1, 0, 0, 0), (3, 3, 2, 1.0, 0, 1, 1, 0, 0), (8, 8, 3, 1.0, 2, 0, 0, 0, 0),
             (9, 17, 4, 1.0, 3, 1, 1, 0, 0), (63, 65, 5, 1.0, 0, 0, 1, 0, 0), (263, 131, 6, 1.5, 2, 0, 2, 1, 0),
             (129, 97, 7, 1.0, 1, 0, 1, 0, 0), (200, 264, 8, 0.7, 3, 0, 3, 0, 1), (300, 280, 9, 1.0, 2, 1, 1, 0, 0),
             (520, 512, 10, 1.0, 1, 1, 3, 0, 0), (96, 80, 11, 1.0, 1, 1, 1, 0, 2), (96, 80, 12, 1.0, 2, 1, 1, 0, 3),
             (96, 80, 13, 1.0, 1, 1, 1, 0, 4), (96, 80, 14, 1.0, 2, 0, 1, 0, 5), (96, 80, 15, 1.0, 1, 1, 1, 0, 6),
             (96, 80, 16, 1.0, 1, 1, 1, 0, 7)]
# The output formats stage C is checked in on the oracle (XYB_F32_PLANAR is the stage-B tap)
FORMATS = [abi.FORMAT_RGB_F32, abi.FORMAT_RGB_U8, abi.FORMAT_RGBA_U8, abi.FORMAT_RGB_U16, abi.FORMAT_RGB_F16]


def _case_id(c):
    return f"{c[0]}x{c[1]}-epf{c[4]}-gab{c[5]}-p{c[6]}-colour{c[8]}"


def _read(name):
    import os
    return open(os.path.join(fp.ROOT, GOLDEN, name + ".jxl"), "rb").read()


def _synthetic(case):
    import synth
    w, h, seed, dist, epf, gab, profile, entropy, colour = case
    return synth.encode_synthetic(w, h, seed, dist, epf, gab, profile, entropy=entropy, colour=colour)


def _frame(data, fmt=abi.FORMAT_RGB_F32):
    import jxl_rs_b200 as j
    pf = j.ParsedFrame(data)
    d, *_ = pf.desc(fmt)
    return fp.Frame(d)


def _check_file(data, what):
    from tests import oracle_binding as ob
    fr = _frame(data)
    out, taps = ob.decode_file(data, abi.FORMAT_RGB_F32, taps=True)
    a, ma = fp.stage_a(fr, taps["coeffs"])
    ratios = [fp.check("A", taps["xyb_idct"], a, ma, what)]
    b, mb = fp.stage_b(fr, taps["xyb_idct"].astype(np.float64))
    ratios.append(fp.check("B", taps["xyb_filtered"], b, mb, what))
    ratios.append(_check_outputs(data, None, taps["xyb_filtered"], what, {abi.FORMAT_RGB_F32: out}))
    return ratios


def _check_outputs(data, fr, xyb, what, have=None):
    """fr: an edited frame descriptor used for every format, or None for the file's own (per format). Every output format of the oracle against stage C of its own filtered planes, in display orientation; the
    oracle is also allowed its fast_powf / fast_log2f error (3e-5 relative) for gamma and HLG. RGBA must equal the
    RGB_U8 output byte for byte, with alpha 255. Returns the largest err / (2^-24 M) of the f32 output."""
    from tests import oracle_binding as ob
    outs = dict(have or {})
    ratio, refs = 0.0, {}
    for fmt in FORMATS:
        if fmt not in outs:
            outs[fmt], _ = ob.decode_file(data, fmt)
        ff = _frame(data, fmt) if fr is None else fr  # the output curve can depend on the format (float: linear)
        key = (ff.output_tf, ff.output_gamma, ff.intensity_target)
        if key not in refs:
            refs[key] = fp.stage_c(ff, xyb.astype(np.float64), full=True)
        c, mc, allow, _ = refs[key]
        r = fp.check_output(fmt, outs[fmt], c, mc, ff.output_tf, ff.orientation, what, allow)
        ratio = r if fmt == abi.FORMAT_RGB_F32 else ratio
    assert np.array_equal(outs[abi.FORMAT_RGBA_U8][..., :3], outs[abi.FORMAT_RGB_U8]), f"{what}: RGBA colour != RGB_U8"
    return ratio


@pytest.mark.parametrize("case", SYNTHETIC, ids=[_case_id(c) for c in SYNTHETIC])
def test_synthetic_frames_match_f64(case):
    _check_file(_synthetic(case), str(case))


@pytest.mark.parametrize("name", FIXTURES)
def test_fixtures_match_f64(name):
    _check_file(_read(name), name)


def test_afv_basis_is_orthonormal():
    """The AFV 4x4 basis (transform.rs:34-291) is an orthonormal 16x16 matrix: a mistyped constant breaks it."""
    b = fp.AFV_BASIS
    assert np.abs(b @ b.T - np.eye(16)).max() < 1e-6


@pytest.mark.parametrize("t", range(27))
def test_transform_to_pixels_matches_f64(t):
    """jxo_transform_to_pixels against the f64 definition of each of the 27 transform types: random coefficients with
    exact zeros, a few large values and random LF samples."""
    from tests import oracle_binding as ob
    lib = ob.load()
    cx, cy = fp.COV_X[t], fp.COV_Y[t]
    n = 64 * cx * cy
    rng = np.random.default_rng(100 + t)
    reps = 8 if n <= 1024 else 2
    for r in range(reps):
        co = rng.normal(0, 0.05, n) * (rng.random(n) < 0.6)
        co[rng.integers(0, n, 3)] = rng.choice([-40.0, 25.0, 300.0], 3)
        if r == 0:
            co[:] = 0.0
        lf = rng.normal(0, 1.0, (cy, cx))
        co32, lf32 = co.astype(np.float32), lf.astype(np.float32)
        buf = co32.copy()
        l32 = lf32.reshape(-1).copy()
        lib.jxo_transform_to_pixels(t, l32.ctypes.data, buf.ctypes.data)
        c64, l64 = co32.astype(np.float64)[None], lf32.astype(np.float64)[None]
        want, mag = fp.transform_to_pixels_batch(t, c64, l64, np.abs(c64), np.abs(l64))
        fp.check("A", buf.reshape(8 * cy, 8 * cx), want[0], mag[0], f"type {t}")


# ---------------------------------------------------------------------------------------------------------------------
# Sensitivity: one planted fault on the f64 side must fail the bound
# ---------------------------------------------------------------------------------------------------------------------
def _stage_a_fails(data, fr=None):
    from tests import oracle_binding as ob
    fr = fr or _frame(data)
    _, taps = ob.decode_file(data, abi.FORMAT_RGB_F32, taps=True)
    a, ma = fp.stage_a(fr, taps["coeffs"])
    with pytest.raises(AssertionError):
        fp.check("A", taps["xyb_idct"], a, ma)


def _stage_b_fails(data, fr=None, taps=None):
    from tests import oracle_binding as ob
    fr = fr or _frame(data)
    if taps is None:
        _, taps = ob.decode_file(data, abi.FORMAT_RGB_F32, taps=True)
    b, mb = fp.stage_b(fr, taps["xyb_idct"].astype(np.float64))
    with pytest.raises(AssertionError):
        fp.check("B", taps["xyb_filtered"], b, mb)


def test_fault_afv_basis_entry(monkeypatch):
    """One AFV basis entry off by 1e-4. Old abs-or-rel 1e-3 bar on the same planes: not caught (largest difference
    7.9e-5)."""
    basis = fp.AFV_BASIS.copy()
    basis[5, 6] += 1e-4
    monkeypatch.setattr(fp, "AFV_BASIS", basis)
    _stage_a_fails(_read("dice"))


def test_fault_transposed_dequant_matrix():
    """The dequantisation matrix of DCT16X8 read transposed (16x8 instead of 8x16). Old abs-or-rel 1e-3 bar on the
    same planes: caught (largest difference 3.7e-2)."""
    data = _synthetic((300, 280, 9, 1.0, 2, 1, 1, 0, 0))
    fr = _frame(data)
    assert (fr.transform_map == 128 | 6).any()
    fr.dequant[6] = tuple(m.reshape(3, 8, 16).transpose(0, 2, 1).reshape(3, 128) for m in fp.dequant_table(6))
    _stage_a_fails(data, fr)


def test_fault_cfl_tile_off_by_one(monkeypatch):
    """Chroma-from-luma factors taken from the tile one block further on (wrong at every 64-pixel boundary). Old
    abs-or-rel 1e-3 bar on the same planes: caught (largest difference 1.1e-2)."""
    monkeypatch.setattr(fp, "cfl_tile", lambda b: (b + 1) // fp.COLOR_TILE_BLOCKS)
    _stage_a_fails(_synthetic((300, 280, 9, 1.0, 2, 1, 1, 0, 0)))


def test_fault_epf_border_on_wrong_rows(monkeypatch):
    """epf_border_sad_mul applied one pixel off the 8x8 block border. Old abs-or-rel 1e-3 bar on the same planes:
    caught (largest difference 4.4e-3)."""
    monkeypatch.setattr(fp, "epf_border", lambda ys, xs: np.isin((ys + 1) % 8, (0, 7)) | np.isin((xs + 1) % 8, (0, 7)))
    _stage_b_fails(_read("green_queen_vardct_e3"))


def test_fault_mirroring_at_padded_edge(monkeypatch):
    """Filters mirrored at the edge of the planes padded to whole blocks instead of the coded edge (63x65 frame,
    Gaborish + EPF 3). Old abs-or-rel 1e-3 bar on the same planes: caught, narrowly (largest difference 1.4e-3)."""
    monkeypatch.setattr(fp, "filter_input", lambda planes, w, h: planes)
    _stage_b_fails(_synthetic((63, 65, 5, 1.0, 3, 1, 1, 0, 0)))


def test_fault_gaborish_weights_of_x_and_b_swapped():
    """Every available frame carries the default Gaborish weights, equal in all channels, so the frame is decoded by the
    oracle with distinct X / Y / B weights written into its descriptor; swapping X and B on the f64 side must fail.
    Old abs-or-rel 1e-3 bar on the same planes: caught (largest difference 1.1e-2)."""
    import jxl_rs_b200 as j
    from tests import oracle_binding as ob
    data = _synthetic((129, 97, 7, 1.0, 0, 1, 1, 0, 0))
    pf = j.ParsedFrame(data)
    d, hf, off, ln, n = pf.desc(abi.FORMAT_XYB_F32_PLANAR)
    d.gab, d.epf_iters = 1, 0
    for c, (w1, w2) in enumerate([(0.09, 0.05), (0.115169525, 0.061248592), (0.14, 0.075)]):
        d.gab_w1[c], d.gab_w2[c] = w1, w2
    fr = fp.Frame(d)
    ps, pr = fr.xb * 8, fr.yb * 8
    taps = {"coeffs": np.zeros((pf.info.num_groups, 3, 65536), np.int32), "xyb_idct": np.zeros((3, pr, ps), np.float32),
            "xyb_filtered": np.zeros((3, fr.height, fr.width), np.float32)}
    t = ob.JxoTaps(taps["coeffs"].ctypes.data, taps["xyb_idct"].ctypes.data, taps["xyb_filtered"].ctypes.data)
    bad = C.c_uint32()
    assert ob.load().jxo_decode_frame(C.byref(d), hf, off, ln, n, None, 0, C.byref(t), 1, C.byref(bad)) == 0
    b, mb = fp.stage_b(fr, taps["xyb_idct"].astype(np.float64))
    fp.check("B", taps["xyb_filtered"], b, mb)  # the distinct weights themselves are followed
    fr.gab_w1, fr.gab_w2 = fr.gab_w1[[2, 1, 0]], fr.gab_w2[[2, 1, 0]]
    _stage_b_fails(data, fr, taps)


# ---------------------------------------------------------------------------------------------------------------------
# Output stage: stores, curves and edge values
# ---------------------------------------------------------------------------------------------------------------------
def _f16_sweep():
    """Every f32 exponent, both signs, with mantissas that hit ties, round-up carries and the subnormal truncation."""
    rng = np.random.default_rng(7)
    exps = np.arange(256, dtype=np.uint32)
    mants = np.concatenate([np.array([0, 1, 0x1000, 0x1001, 0x2000, 0x3000, 0x7FF000, 0x7FFFFF, 0x7FEFFF], np.uint32),
                            rng.integers(0, 1 << 23, 48, dtype=np.uint32)])
    bits = (exps[:, None] << 23 | mants[None, :]).reshape(-1)
    bits = np.concatenate([bits, bits | np.uint32(0x80000000)])
    return bits.view(np.float32)


def test_f16_restatement_matches_oracle_conversion():
    """f64_pipeline.f16_from_f32 (float16.rs:82-141 in numpy) against the oracle's f32 -> f16 conversion on a dense
    sweep of every exponent; NaN payloads aside the codes must be equal."""
    from tests import oracle_binding as ob
    v = _f16_sweep()
    want = np.zeros(v.size, np.uint16)
    ob.load().jxo_f32_to_f16(C.c_int(v.size), C.c_void_p(v.ctypes.data), C.c_void_p(want.ctypes.data))
    got = fp.f16_from_f32(v)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5].tolist()
    sub = (np.abs(v) >= 2.0 ** -15) & (np.abs(v) < 2.0 ** -14)
    assert sub.any() and np.all(fp.f16_value(got[sub]) <= np.abs(v[sub]) / 2)  # the reference's extra one-bit shift


def _edge_frame(curve_edits, orientation=1):
    """The 256x128 Gaborish + EPF 2, DCT8-only frame with its LF overwritten by the edge targets; returns a function
    decoding it on the oracle in a given format (output, taps) and the edited f64 frame."""
    import jxl_rs_b200 as j
    from tests import oracle_binding as ob
    pf = j.ParsedFrame(_synthetic((256, 128, 5, 4.0, 2, 1, 0, 0, 0)))
    fr0 = fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0])
    lf = fp.edge_lf(fr0, fp.edge_targets(), curve_edits["intensity_target"])
    keep = []

    def decode(fmt):
        d, hf, off, ln, n = pf.desc(fmt)
        fp.edit_desc(d, lf, orientation=orientation, **curve_edits)
        fr = fp.Frame(d)
        h, w = (fr.width, fr.height) if orientation >= 5 else (fr.height, fr.width)
        ch = 4 if fmt == abi.FORMAT_RGBA_U8 else 3
        dt = {abi.FORMAT_RGB_F32: np.float32, abi.FORMAT_RGB_U16: np.uint16, abi.FORMAT_RGB_F16: np.uint16}.get(fmt, np.uint8)
        out = np.zeros((h, w, ch), dt)
        taps = {"coeffs": np.zeros((pf.info.num_groups, 3, 65536), np.int32),
                "xyb_idct": np.zeros((3, fr.yb * 8, fr.xb * 8), np.float32),
                "xyb_filtered": np.zeros((3, fr.height, fr.width), np.float32)}
        t = ob.JxoTaps(taps["coeffs"].ctypes.data, taps["xyb_idct"].ctypes.data, taps["xyb_filtered"].ctypes.data)
        bad = C.c_uint32()
        assert ob.load().jxo_decode_frame(C.byref(d), hf, off, ln, n, out.ctypes.data, out.strides[0], C.byref(t), 1,
                                          C.byref(bad)) == 0
        keep.append(d)
        return out, taps, fr
    return decode


EDGE_CURVES = [("linear", fp.TF_LINEAR, 1.0, 255.0), ("srgb", fp.TF_SRGB, 1.0, 255.0), ("gamma2.2", fp.TF_GAMMA, 1 / 2.2, 255.0),
               ("dci", fp.TF_GAMMA, 1 / 2.6, 255.0), ("bt709", fp.TF_BT709, 1.0, 255.0), ("pq", fp.TF_PQ, 1.0, 1000.0),
               ("hlg1000", fp.TF_HLG, 1.0, 1000.0), ("hlg100", fp.TF_HLG, 1.0, 100.0)]


def _edits(curve):
    return {"output_tf": curve[1], "output_gamma": curve[2], "intensity_target": curve[3],
            "output_luminances": fp.BT2100_LUMINANCES}


@pytest.mark.parametrize("curve", EDGE_CURVES, ids=[c[0] for c in EDGE_CURVES])
def test_edge_value_frames_match_f64_on_oracle(curve):
    """The edge-value frame (f64_pipeline.edge_targets) through stages A, B and C of the oracle, in every format, at the
    oracle's bar (f32 bound plus 3e-5 relative on fast_powf / fast_log2f). For HLG this holds the oracle to the +256
    rule of fast_log2f on negative mixed luminances. Every edge region must hold samples."""
    decode = _edge_frame(_edits(curve))
    out, taps, fr = decode(abi.FORMAT_RGB_F32)
    a, ma = fp.stage_a(fr, taps["coeffs"])
    fp.check("A", taps["xyb_idct"], a, ma, curve[0])
    b, mb = fp.stage_b(fr, taps["xyb_idct"].astype(np.float64))
    fp.check("B", taps["xyb_filtered"], b, mb, curve[0])
    xyb = taps["xyb_filtered"].astype(np.float64)
    c, mc, allow, amb = fp.stage_c(fr, xyb, full=True)
    fp.check("C", out, c, mc, curve[0], allow)
    for fmt in (abi.FORMAT_RGB_U8, abi.FORMAT_RGBA_U8, abi.FORMAT_RGB_U16, abi.FORMAT_RGB_F16):
        got, _, _ = decode(fmt)
        fp.check_output(fmt, got, c, mc, fr.output_tf, 1, f"{curve[0]} format {fmt}", allow)
    counts = fp.edge_regions(fp.linear_rgb_f64(fr, xyb), c, fr.output_tf, fp.BT2100_LUMINANCES)
    empty = [k for k, v in counts.items() if v == 0 and not (k == "f16_subnormal" and curve[0] in fp.NO_F16_SUBNORMALS)]
    assert not empty, f"{curve[0]}: empty edge regions {empty} ({counts})"
    if fr.output_tf == fp.TF_HLG:
        assert int(amb.sum()) < amb.size // 8, "too many samples with an undetermined sign of the mixed luminance"


@pytest.mark.parametrize("orientation", range(1, 9))
def test_oracle_orientation_matches_f64(orientation):
    """The oracle's save stage at every orientation and format against orient(stage C) (interval rule)."""
    decode = _edge_frame(_edits(EDGE_CURVES[1]), orientation)
    _, taps, fr = decode(abi.FORMAT_RGB_F32)
    c, mc = fp.stage_c(fr, taps["xyb_filtered"].astype(np.float64))
    for fmt in FORMATS:
        got, _, _ = decode(fmt)
        fp.check_output(fmt, got, c, mc, fr.output_tf, orientation, f"orientation {orientation} format {fmt}")


# Sensitivity of the output-stage checks: one planted fault each, on the f64 side, must fail.
def _oracle_edge(curve, fmt, orientation=1):
    decode = _edge_frame(_edits(curve), orientation)
    _, taps, fr = decode(abi.FORMAT_RGB_F32)
    got, _, _ = decode(fmt)
    return got, taps["xyb_filtered"].astype(np.float64), fr


def test_fault_f16_ieee_subnormals(monkeypatch):
    """f16 stores rounding into the subnormal range like IEEE instead of the reference's truncation with its extra
    one-bit shift. Old bar (1e-3 + 2^-11 against the oracle): not caught (the largest change is 2^-15)."""
    got, xyb, fr = _oracle_edge(EDGE_CURVES[0], abi.FORMAT_RGB_F16)
    c, mc = fp.stage_c(fr, xyb)
    fp.check_output(fp.FMT_F16, got, c, mc, fr.output_tf)
    monkeypatch.setattr(fp, "f16_from_f32", lambda v: np.asarray(v, np.float32).astype(np.float16).view(np.uint16))
    with pytest.raises(AssertionError):
        fp.check_output(fp.FMT_F16, got, c, mc, fr.output_tf)


def test_fault_u16_truncated():
    """u16 codes truncated instead of rounded. Old bar (64 LSB against the oracle): not caught (1 LSB)."""
    got, xyb, fr = _oracle_edge(EDGE_CURVES[1], abi.FORMAT_RGB_U16)
    c, mc = fp.stage_c(fr, xyb)
    bad = np.floor(np.clip(c, 0, 1) * 65535.0).astype(np.uint16)
    fp.check_output(fp.FMT_U16, got, c, mc, fr.output_tf)
    with pytest.raises(AssertionError):
        fp.check_output(fp.FMT_U16, bad, c, mc, fr.output_tf)


def test_fault_hlg_nan_for_non_positive_mixed():
    """HLG with log2 of a non-positive mixed luminance (NaN) instead of the fast_log2f rule, as the CUDA kernel computed
    it before. Old bars: the u8 output agrees by accident (NaN stores as 0); no check looked at f32 or f16 there."""
    got, xyb, fr = _oracle_edge(EDGE_CURVES[6], abi.FORMAT_RGB_F32)
    c, mc, allow, _ = fp.stage_c(fr, xyb, full=True)
    lin = fp.linear_rgb_f64(fr, xyb)
    mixed = lin @ np.asarray(fp.BT2100_LUMINANCES)
    planted = got.copy()
    planted[mixed <= 0] = np.nan
    assert (mixed <= 0).any()
    with pytest.raises(AssertionError):
        fp.check("C", planted, c, mc, "planted", allow)


def test_fault_gamma_exponent_off(monkeypatch):
    """The gamma exponent off by 1e-4 on the f64 side. Old bar (oracle within 1e-3): not caught (about 2e-4)."""
    got, xyb, fr = _oracle_edge(EDGE_CURVES[2], abi.FORMAT_RGB_F32)
    c, mc, allow, _ = fp.stage_c(fr, xyb, full=True)
    fp.check("C", got, c, mc, "gamma", allow)
    fr.output_gamma += 1e-4
    c, mc, allow, _ = fp.stage_c(fr, xyb, full=True)
    with pytest.raises(AssertionError):
        fp.check("C", got, c, mc, "gamma", allow)


def test_fault_orientations_5_and_7_swapped(monkeypatch):
    """orient with orientations 5 and 7 exchanged. Old bar (1 LSB against the oracle): caught for u8, but only as a
    whole-image mismatch; here the f64 interval rule fails on its own."""
    got, xyb, fr = _oracle_edge(EDGE_CURVES[1], abi.FORMAT_RGB_U8, orientation=5)
    c, mc = fp.stage_c(fr, xyb)
    fp.check_output(fp.FMT_U8, got, c, mc, fr.output_tf, 5)
    orig = fp.orient
    monkeypatch.setattr(fp, "orient", lambda img, o: orig(img, {5: 7, 7: 5}.get(o, o)))
    with pytest.raises(AssertionError):
        fp.check_output(fp.FMT_U8, got, c, mc, fr.output_tf, 5)


def test_fault_alpha_254():
    """RGBA with alpha 254. Old bar (1 LSB against the oracle's RGBA): not caught."""
    got, xyb, fr = _oracle_edge(EDGE_CURVES[1], abi.FORMAT_RGBA_U8)
    c, mc = fp.stage_c(fr, xyb)
    fp.check_output(fp.FMT_RGBA_U8, got, c, mc, fr.output_tf)
    got = got.copy()
    got[..., 3] = 254
    with pytest.raises(AssertionError):
        fp.check_output(fp.FMT_RGBA_U8, got, c, mc, fr.output_tf)
