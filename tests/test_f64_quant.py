"""Dequantisation matrices against the float64 restatement of quant_weights.rs in tests/f64_quant.py: the library
tables in every entry, custom tables of every mode the reference permits at every table index (written by the
synthetic writer and read back by the front-end), the reference's refusals, stage A of the oracle on frames with custom
tables, and planted faults the bound |got - ref| <= K_q 2^-24 M must catch. No GPU."""
import ctypes as C

import numpy as np
import pytest

import jxl_rs_b200 as j
from jxl_rs_b200 import abi
from tests import f64_pipeline as fp
from tests import f64_quant as fq

PAIRS = [(idx, mode) for idx in range(17) for mode in fq.permitted_modes(idx)]
BAND_MODES = (fq.MODE_DCT4, fq.MODE_DCT4X8, fq.MODE_AFV, fq.MODE_DCT)


def _encode(dequant, w=8, h=8, seed=1, profile=0, x_qm_scale=3, b_qm_scale=2):
    import synth
    return synth.encode_synthetic(w, h, seed, 1.0, 2, 1, profile, dequant=dequant, x_qm_scale=x_qm_scale,
                                  b_qm_scale=b_qm_scale)


def _parse(data):
    """(ParsedFrame, descriptor): the descriptor's arrays live as long as the ParsedFrame."""
    pf = j.ParsedFrame(data)
    return pf, pf.desc(abi.FORMAT_RGB_F32)[0]


def _one(idx, enc):
    dq = [None] * 17
    dq[idx] = enc
    return dq


def frontend_table(d, idx):
    """The front-end's custom table idx of a parsed frame (desc.dequant_tables[idx]) as (3, num) float32."""
    n = fq.num_entries(idx)
    assert d.dequant_tables[idx], f"table {idx} is not custom in the frame"
    return np.ctypeslib.as_array(C.cast(d.dequant_tables[idx], C.POINTER(C.c_float)), (3 * n,)).reshape(3, n).copy()


def library_table(idx):
    """The front-end's library table idx through jxo_t_dequant_table, (3, num) float32."""
    from tests import oracle_binding as ob
    lib = ob.load()
    lib.jxo_t_dequant_table.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    lib.jxo_t_dequant_table.restype = C.c_uint32
    n = fq.num_entries(idx)
    out = np.zeros((3, n), np.float32)
    for c in range(3):
        assert lib.jxo_t_dequant_table(fq.TABLE_OF_TRANSFORM.index(idx), c, out[c].ctypes.data, n) == n
    return out


def _custom_cases():
    """(idx, mode, num_bands, seed): every permitted pair; the modes with distance bands at 16 bands (the far corner
    entry is then the closest to the zero band) and at a random count; DCT also at 1 band."""
    cases = []
    for idx, mode in PAIRS:
        if mode in BAND_MODES:
            cases += [(idx, mode, 16, 0), (idx, mode, None, 1)]
            if mode == fq.MODE_DCT:
                cases.append((idx, mode, 1, 2))
        else:
            cases.append((idx, mode, None, 0))
    return cases


CUSTOM = _custom_cases()


@pytest.mark.parametrize("idx", range(17))
def test_library_tables_match_f64(idx):
    """Every entry of all three channels of library table idx, and its size 64 REQUIRED_SIZE_X REQUIRED_SIZE_Y."""
    got = library_table(idx)
    ref, mag = fq.compute_table(fq.library_encoding(idx), idx)
    assert got.shape == ref.shape == (3, 64 * fq.REQUIRED_SIZE_X[idx] * fq.REQUIRED_SIZE_Y[idx])
    fq.check_table(got, ref, mag, f"library table {idx}")


@pytest.mark.parametrize("case", CUSTOM, ids=[f"t{c[0]}-mode{c[1]}-bands{c[2]}-s{c[3]}" for c in CUSTOM])
def test_custom_tables_match_f64(case):
    """A random valid encoding of one (table index, mode) pair, written into a frame whose other tables stay library:
    the front-end's table against the restatement, every entry."""
    idx, mode, nb, seed = case
    enc = fq.random_encoding(np.random.default_rng(1000 * idx + 10 * mode + seed), idx, mode, nb)
    pf, d = _parse(_encode(_one(idx, enc)))
    assert [bool(d.dequant_tables[i]) for i in range(17)] == [i == idx for i in range(17)]
    ref, mag = fq.compute_table(enc, idx)
    fq.check_table(frontend_table(d, idx), ref, mag, f"table {idx} mode {mode}")


def test_every_custom_table_of_one_frame():
    """All 17 tables custom in one frame (RAW on the non-square 6 and 12, DCT on the others, AFV at 10): each read at
    its own index."""
    rng = np.random.default_rng(5)
    modes = {6: fq.MODE_RAW, 12: fq.MODE_RAW, 10: fq.MODE_AFV, 1: fq.MODE_IDENTITY, 2: fq.MODE_DCT2, 3: fq.MODE_DCT4,
             9: fq.MODE_DCT4X8}
    encs = [fq.random_encoding(rng, i, modes.get(i, fq.MODE_DCT)) for i in range(17)]
    pf, d = _parse(_encode(encs))
    for i in range(17):
        ref, mag = fq.compute_table(encs[i], i)
        fq.check_table(frontend_table(d, i), ref, mag, f"table {i}")


# ---------------------------------------------------------------------------------------------------------------------
# Stage A of the oracle on frames with custom tables
# ---------------------------------------------------------------------------------------------------------------------
# (width, height, seed, profile, x_qm_scale, b_qm_scale, encodings seed): profile 4 at 512x512 seed 14 places a
# varblock of every table index
ORACLE_CASES = [(512, 512, 14, 4, 3, 2, 1), (512, 512, 14, 4, 0, 7, 2), (512, 512, 14, 4, 7, 0, 3),
                (200, 136, 3, 1, 0, 0, 4), (96, 80, 5, 0, 7, 7, 5)]


@pytest.mark.parametrize("case", ORACLE_CASES, ids=[f"{c[0]}x{c[1]}-p{c[3]}-xqm{c[4]}-bqm{c[5]}" for c in ORACLE_CASES])
def test_oracle_stage_a_with_custom_tables(case):
    """The oracle's stage A (and B on top) against f64 stage A built from the encodings the frame was written with.
    Every custom table must be read by a varblock of the frame."""
    from tests import oracle_binding as ob
    w, h, seed, profile, xq, bq, es = case
    encs = fq.profile4_encodings(es)
    data = _encode(encs, w, h, seed, profile, xq, bq)
    pf, d = _parse(data)
    assert (int(d.x_qm_scale), int(d.b_qm_scale)) == (xq, bq)
    fr = fp.Frame(d, encodings=encs)
    if profile == 4:
        fq.assert_custom_tables_used(fr, encs, str(case))
    else:
        fr.encodings = encs = [e if i in fq.tables_used(fr) else None for i, e in enumerate(encs)]
        data = _encode(encs, w, h, seed, profile, xq, bq)
        pf, d = _parse(data)
        fr = fp.Frame(d, encodings=encs)
    _, taps = ob.decode_file(data, abi.FORMAT_RGB_F32, taps=True)
    a, ma = fp.stage_a(fr, taps["coeffs"])
    r = fp.check("A", taps["xyb_idct"], a, ma, str(case))
    b, mb = fp.stage_b(fr, taps["xyb_idct"].astype(np.float64))
    fp.check("B", taps["xyb_filtered"], b, mb, str(case))
    print(case, "stage A largest err/(2^-24 M):", round(r, 2))


def test_frame_refuses_missing_encodings():
    """A descriptor with custom tables and no encodings cannot fall back to the front-end's tables."""
    pf, d = _parse(_encode(fq.profile4_encodings(9)))
    with pytest.raises(ValueError):
        fp.Frame(d)
    with pytest.raises(ValueError):
        fp.Frame(d, encodings=[None] * 17)


# ---------------------------------------------------------------------------------------------------------------------
# Refusals: each of the reference's errors must make parsing fail, and the restatement must refuse too
# ---------------------------------------------------------------------------------------------------------------------
H = fq.f16_bits
INF, NAN, ZERO, NEG_ZERO = 0x7C00, 0x7E00, 0x0000, 0x8000


def _dct(first=100.0, rest=(-0.5, -0.5)):
    return [[int(H(first))] + [int(H(v)) for v in rest] for _ in range(3)]


def _with(base, path, value):
    """A copy of a nested list with one f16 entry replaced."""
    out = [list(r) if isinstance(r, list) else r for r in base]
    c, i = path
    out[c] = list(out[c])
    out[c][i] = value
    return out


def _ident(w=(50.0, 100.0, 100.0)):
    return [[int(H(v)) for v in w] for _ in range(3)]


def _afv():
    return [[int(H(v)) for v in (50.0, 50.0, 4.0, 4.0, 4.0, 6.0, -0.25, -0.25, -0.25)] for _ in range(3)]


def _raw(idx, den=2.0 ** -8, entry=None):
    raw = np.full((3, 8 * fq.REQUIRED_SIZE_Y[idx], 8 * fq.REQUIRED_SIZE_X[idx]), 7, np.int64)
    if entry is not None:
        raw[1, 3, 5] = entry
    return {"mode": fq.MODE_RAW, "den": int(H(den)) if not isinstance(den, int) else den, "raw": raw}


REFUSALS = [
    # modes 1..5 on a table larger than 8x8
    ("identity-on-16x16", 4, {"mode": 1, "w": _ident()}, "InvalidQuantEncoding"),
    ("dct2-on-8x16", 6, {"mode": 2, "w": [[int(H(10.0))] * 6] * 3}, "InvalidQuantEncoding"),
    ("dct4-on-32x32", 5, {"mode": 3, "w": [[int(H(1.0))] * 2] * 3, "dct": _dct()}, "InvalidQuantEncoding"),
    ("dct4x8-on-256x256", 15, {"mode": 4, "w": [int(H(1.0))] * 3, "dct": _dct()}, "InvalidQuantEncoding"),
    ("afv-on-64x64", 11, {"mode": 5, "w": _afv(), "dct": _dct(), "dct4": _dct()}, "InvalidQuantEncoding"),
    # a weight below ALMOST_ZERO in magnitude
    ("identity-weight-zero", 1, {"mode": 1, "w": _with(_ident(), (1, 2), ZERO)}, "HfQuantFactorTooSmall"),
    ("dct2-weight-minus-zero", 2, {"mode": 2, "w": _with([[int(H(10.0))] * 6] * 3, (2, 5), NEG_ZERO)},
     "HfQuantFactorTooSmall"),
    ("dct4-divisor-zero", 3, {"mode": 3, "w": _with([[int(H(1.0))] * 2] * 3, (0, 1), ZERO), "dct": _dct()},
     "HfQuantFactorTooSmall"),
    ("dct4x8-divisor-zero", 9, {"mode": 4, "w": [int(H(1.0)), ZERO, int(H(1.0))], "dct": _dct()},
     "HfQuantFactorTooSmall"),
    # params[c][0] below ALMOST_ZERO
    ("dct-first-band-zero", 0, {"mode": 6, "dct": _with(_dct(), (2, 0), ZERO)}, "HfQuantFactorTooSmall"),
    ("dct-first-band-negative", 7, {"mode": 6, "dct": _with(_dct(), (1, 0), int(H(-3.0)))}, "HfQuantFactorTooSmall"),
    ("afv-4x4-first-band-zero", 10, {"mode": 5, "w": _afv(), "dct": _dct(), "dct4": _with(_dct(), (0, 0), ZERO)},
     "HfQuantFactorTooSmall"),
    # a band falling below ALMOST_ZERO through mult: 6e-8 * 64 / 65505
    ("dct-band-below-almost-zero", 4, {"mode": 6, "dct": _with(_with(_dct(), (1, 0), 0x0001), (1, 1), int(H(-65504.0)))},
     "InvalidDistanceBand"),
    ("afv-band-below-almost-zero", 10, {"mode": 5, "w": _with(_with(_afv(), (2, 5), 0x0001), (2, 7), int(H(-65504.0))),
                                         "dct": _dct(), "dct4": _dct()}, "InvalidDistanceBand"),
    # a final weight outside [ALMOST_ZERO, 1 / ALMOST_ZERO]
    ("dct-weight-above-1e8", 8, {"mode": 6, "dct": _with(_with(_dct(), (0, 0), int(H(60000.0))), (0, 1),
                                                          int(H(60000.0)))}, "InvalidQuantizationTableWeight"),
    ("identity-weight-negative", 1, {"mode": 1, "w": _with(_ident(), (0, 0), int(H(-2.0)))},
     "InvalidQuantizationTableWeight"),
    ("identity-weight-inf", 1, {"mode": 1, "w": _with(_ident(), (2, 1), INF)}, "InvalidQuantizationTableWeight"),
    ("identity-weight-nan", 1, {"mode": 1, "w": _with(_ident(), (1, 0), NAN)}, "InvalidQuantizationTableWeight"),
    ("dct2-weight-nan", 2, {"mode": 2, "w": _with([[int(H(10.0))] * 6] * 3, (0, 3), NAN)},
     "InvalidQuantizationTableWeight"),
    ("dct-first-band-inf", 0, {"mode": 6, "dct": _with(_dct(), (0, 0), INF)}, "InvalidQuantizationTableWeight"),
    ("dct-first-band-nan", 12, {"mode": 6, "dct": _with(_dct(), (2, 0), NAN)}, "InvalidQuantizationTableWeight"),
    ("dct-mult-inf", 13, {"mode": 6, "dct": _with(_dct(), (1, 2), INF)}, "InvalidQuantizationTableWeight"),
    ("dct-mult-nan", 5, {"mode": 6, "dct": _with(_dct(), (0, 1), NAN)}, "InvalidQuantizationTableWeight"),
    ("dct4-divisor-inf", 3, {"mode": 3, "w": _with([[int(H(1.0))] * 2] * 3, (1, 0), INF), "dct": _dct()},
     "InvalidQuantizationTableWeight"),
    ("afv-weight-nan", 10, {"mode": 5, "w": _with(_afv(), (1, 3), NAN), "dct": _dct(), "dct4": _dct()},
     "InvalidQuantizationTableWeight"),
    ("afv-weight-negative", 10, {"mode": 5, "w": _with(_afv(), (0, 0), int(H(-1.0))), "dct": _dct(), "dct4": _dct()},
     "InvalidQuantizationTableWeight"),
    # RAW: a denominator below ALMOST_ZERO, an entry <= 0
    ("raw-den-zero", 0, _raw(0, den=ZERO), "InvalidRawQuantTable"),
    ("raw-den-negative", 6, _raw(6, den=-1.0), "InvalidRawQuantTable"),
    ("raw-entry-zero", 12, _raw(12, entry=0), "InvalidRawQuantTable"),
    ("raw-entry-negative", 4, _raw(4, entry=-5), "InvalidRawQuantTable"),
]


@pytest.mark.parametrize("case", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_refusals(case):
    """Parsing fails with a JxgError (never decodes), and the restatement names the reference's error."""
    name, idx, enc, error = case
    with pytest.raises(fq.Refused, match=error):
        fq.compute_table(enc, idx)
    data = _encode(_one(idx, enc))
    with pytest.raises(j.JxgError):
        j.ParsedFrame(data)


def test_accepted_near_the_limits():
    """The accepting side of the same checks: f16 subnormal weights (>= ALMOST_ZERO) and a RAW entry of 1 parse, and
    their tables match."""
    cases = [(1, {"mode": 1, "w": _with(_ident(), (0, 1), 0x0001)}),
             (0, {"mode": 6, "dct": _with(_dct(), (0, 0), 0x0001)}),
             (6, _raw(6, entry=1))]
    for idx, enc in cases:
        pf, d = _parse(_encode(_one(idx, enc)))
        ref, mag = fq.compute_table(enc, idx)
        fq.check_table(frontend_table(d, idx), ref, mag, f"table {idx}")


# ---------------------------------------------------------------------------------------------------------------------
# Planted faults on the f64 side: the bound must catch each one
# ---------------------------------------------------------------------------------------------------------------------
def _custom_frontend(idx, enc):
    pf, d = _parse(_encode(_one(idx, enc)))
    return frontend_table(d, idx)


def _fails(got, ref, mag):
    with pytest.raises(AssertionError):
        fq.check_table(got, ref, mag)


def test_fault_raw_read_transposed():
    """A RAW table read with x and y swapped (rows 8 REQUIRED_SIZE_Y long instead of 8 REQUIRED_SIZE_X) on the
    non-square table 12 (32x64). Library tables alone would not expose it: no library table is RAW."""
    idx = 12
    enc = fq.random_encoding(np.random.default_rng(3), idx, fq.MODE_RAW)
    got = _custom_frontend(idx, enc)
    fq.check_table(got, *fq.compute_table(enc, idx))
    bad = dict(enc, raw=np.asarray(enc["raw"]).reshape(3, 8 * fq.REQUIRED_SIZE_X[idx], -1).transpose(0, 2, 1))
    _fails(got, *fq.compute_table(bad, idx))


def test_fault_dct4_divisors_swapped(monkeypatch):
    """DCT4's two divisors exchanged (xyb_mul[c][0] on entry 9, xyb_mul[c][1] on entries 1 and 8). Library tables
    alone would not expose it: the library DCT4X4 divisors are all 1."""
    idx = 3
    enc = fq.random_encoding(np.random.default_rng(4), idx, fq.MODE_DCT4)
    got = _custom_frontend(idx, enc)
    fq.check_table(got, *fq.compute_table(enc, idx))
    swapped = {"mode": enc["mode"], "w": np.asarray(enc["w"])[:, ::-1], "dct": enc["dct"]}
    _fails(got, *fq.compute_table(swapped, idx))
    lib = fq.library_encoding(idx)
    fq.check_table(library_table(idx), *fq.compute_table(dict(lib, w=lib["w"][:, ::-1]), idx))  # not exposed


def test_fault_mult_negative_branch(monkeypatch):
    """mult(v) = 1 - v for v <= 0 instead of 1 / (1 - v). Library tables alone would expose it: their band parameters
    are negative."""
    idx = 4
    enc = fq.random_encoding(np.random.default_rng(5), idx, fq.MODE_DCT, 16)
    got = _custom_frontend(idx, enc)
    fq.check_table(got, *fq.compute_table(enc, idx))
    monkeypatch.setattr(fq, "mult", lambda v: 1.0 + v if v > 0 else 1.0 - v)
    _fails(got, *fq.compute_table(enc, idx))
    _fails(library_table(idx), *fq.compute_table(fq.library_encoding(idx), idx))


def test_fault_afv_frequencies_swapped(monkeypatch):
    """Two AFV frequencies exchanged (entries 2 and 7 of FREQS, 0.85 and 5.45). Library tables alone would expose it,
    through B only: the library's X and Y AFV bands are flat (mult(0) = 1), so only B's -0.25 bands see a position."""
    idx = 10
    enc = fq.random_encoding(np.random.default_rng(6), idx, fq.MODE_AFV)
    got = _custom_frontend(idx, enc)
    fq.check_table(got, *fq.compute_table(enc, idx))
    freqs = fq.AFV_FREQS.copy()
    freqs[[2, 7]] = freqs[[7, 2]]
    monkeypatch.setattr(fq, "AFV_FREQS", freqs)
    _fails(got, *fq.compute_table(enc, idx))
    lib_got, (lib_ref, lib_mag) = library_table(idx), fq.compute_table(fq.library_encoding(idx), idx)
    fq.check_table(lib_got[:2], lib_ref[:2], lib_mag[:2])  # X and Y do not see it
    _fails(lib_got[2:], lib_ref[2:], lib_mag[2:])


def test_fault_x_and_b_tables_swapped():
    """The X and B channels of a table exchanged. Library tables alone would expose it (their X and B differ)."""
    idx = 7
    enc = fq.random_encoding(np.random.default_rng(7), idx, fq.MODE_DCT, 16)
    got = _custom_frontend(idx, enc)
    ref, mag = fq.compute_table(enc, idx)
    fq.check_table(got, ref, mag)
    _fails(got, ref[[2, 1, 0]], mag[[2, 1, 0]])


def test_fault_one_entry_of_256x256_off():
    """One entry of the 256x256 table (index 15) off by 1e-4 relative, in the front-end's table. Library tables
    alone expose it only with every entry checked: the reference's sampled known answers see about one entry in ten."""
    idx = 15
    enc = fq.random_encoding(np.random.default_rng(8), idx, fq.MODE_DCT, 16)
    got = _custom_frontend(idx, enc)
    ref, mag = fq.compute_table(enc, idx)
    fq.check_table(got, ref, mag)
    for table, (r, m) in ((got, (ref, mag)), (library_table(idx), fq.compute_table(fq.library_encoding(idx), idx))):
        bad = table.copy()
        bad[1, 40000] *= 1.0 + 1e-4
        _fails(bad, r, m)
