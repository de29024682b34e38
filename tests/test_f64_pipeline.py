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
# Outputs whose curve stage C does not restate (gamma: fixtures 3x3*, colour 2 and 7; HLG: colour 4): f64_pipeline
# explains why. Listed here so that a case cannot lose its stage-C check unnoticed.
NO_STAGE_C = {"3x3_srgb_lossy", "3x3a_srgb_lossy", "colour2", "colour4", "colour7"}


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


def _check_file(data, what, stage_c=True):
    from tests import oracle_binding as ob
    fr = _frame(data)
    out, taps = ob.decode_file(data, abi.FORMAT_RGB_F32, taps=True)
    a, ma = fp.stage_a(fr, taps["coeffs"])
    ratios = [fp.check("A", taps["xyb_idct"], a, ma, what)]
    b, mb = fp.stage_b(fr, taps["xyb_idct"].astype(np.float64))
    ratios.append(fp.check("B", taps["xyb_filtered"], b, mb, what))
    if not stage_c:
        assert fr.output_tf not in fp.SUPPORTED_TF, f"{what}: stage C is restated for this output, check it"
        return ratios
    c, mc = fp.stage_c(fr, taps["xyb_filtered"].astype(np.float64))
    ratios.append(fp.check("C", out, c, mc, what))
    fr8 = _frame(data, abi.FORMAT_RGB_U8)
    c8, mc8 = fp.stage_c(fr8, taps["xyb_filtered"].astype(np.float64))
    u8, _ = ob.decode_file(data, abi.FORMAT_RGB_U8)
    fp.check_u8(u8, fp.u8_store_f64(c8), mc8, what)
    return ratios


@pytest.mark.parametrize("case", SYNTHETIC, ids=[_case_id(c) for c in SYNTHETIC])
def test_synthetic_frames_match_f64(case):
    _check_file(_synthetic(case), str(case), stage_c=f"colour{case[8]}" not in NO_STAGE_C)


@pytest.mark.parametrize("name", FIXTURES)
def test_fixtures_match_f64(name):
    _check_file(_read(name), name, stage_c=name not in NO_STAGE_C)


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
    fr.dequant[6] = fp.dequant_table(6).reshape(3, 8, 16).transpose(0, 2, 1).reshape(3, 128)
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
