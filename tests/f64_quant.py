"""Float64 restatement of the dequantisation matrices, written from the reference text jxl/src/frame/quant_weights.rs
(not a test module).

Encodings are plain Python values. A custom encoding, as a frame's HfGlobal carries it, is a dict with "mode" 1..7 and
its parameters as f16 BIT PATTERNS, so that they decode exactly and invalid values (zero, negative, inf, NaN) can be
written down:

  1 Identity  {"w": 3 x 3}                     2 DCT2   {"w": 3 x 6}
  3 DCT4      {"w": 3 x 2 (xyb_mul), "dct"}    4 DCT4X8 {"w": 3 (xyb_mul), "dct"}
  5 AFV       {"w": 3 x 9, "dct" (4x8), "dct4" (4x4)}
  6 DCT       {"dct"}                          7 RAW    {"den": f16, "raw": 3 x (8 REQUIRED_SIZE_Y) x (8 REQUIRED_SIZE_X)
                                                          ints, each channel in raster order, 8 REQUIRED_SIZE_X wide}
  "dct" / "dct4": 3 rows of num_bands (1..16) f16 values (DctQuantWeightParams).

library_encoding(idx) gives the library default of a table index with float values (marked "library"); its parameter
literals are read from jxl_rs_b200/csrc/host/quant_params.inc as data, each literal and product rounded to f32 as the
reference's f32 constants are. The reference's own known answers (test_kat_entropy.py) pin those literals.

compute_table(enc, idx) returns the table (3, 64 REQUIRED_SIZE_X REQUIRED_SIZE_Y) in float64 and a magnitude M per entry,
or raises Refused where the reference returns an error. An f32 implementation meets |got - table| <= K_Q 2^-24 M.

M. Every weight is a product of f32 roundings, each at most 2^-24 relative, so the error of a table entry T = 1 / w is
a multiple of 2^-24 |T|. M = |T| (1 + i + |ln(b / a)| s) for an interpolated entry, |T| for a direct one:
  - 1: the final 1 / w and the few single roundings of a direct entry (x 64 is exact; DCT4 / DCT4X8 divide once more).
  - i: band i = bands[0] * mult(p_1) * ... * mult(p_i) carries i products and i mult roundings; a = band i and
    b = band i + 1 both enter (b / a)^frac * a.
  - |ln(b / a)| s: the scaled distance s = sqrt(dx^2 + dy^2) (the powf exponent is its fractional part) has a relative
    error of a few roundings (scale, rcp, x * rcp, squares, sqrt); an absolute error e s in the exponent changes
    (b / a)^frac by the factor exp(|ln(b / a)| e s). The AFV bands interpolate the same way in pos * 3 / max.
  powf, sqrt and the divisions add a few ulps more; they and the constant factors go into K_Q, set at four times the
  largest ratio measured on the front-end (DESIGN.md section 4).
"""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 2.0 ** -24
K_Q = 16  # four times the largest err / (2^-24 M) of the front-end's tables, rounded up; DESIGN.md section 4

F32 = np.float32
ALMOST_ZERO = float(F32(1e-8))                                  # quant_weights.rs:32
MAX_WEIGHT = float(F32(1.0) / F32(1e-8))                        # 1 / ALMOST_ZERO, in f32
REQUIRED_SIZE_X = [1, 1, 1, 1, 2, 4, 1, 1, 2, 1, 1, 8, 4, 16, 8, 32, 16]  # quant_weights.rs:1128-1132
REQUIRED_SIZE_Y = [1, 1, 1, 1, 2, 4, 2, 4, 4, 1, 1, 8, 8, 16, 16, 32, 32]
TABLE_OF_TRANSFORM = [0, 1, 2, 3, 4, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 10, 10, 11, 12, 12, 13, 14, 14, 15, 16, 16]  # :321-343
MODE_IDENTITY, MODE_DCT2, MODE_DCT4, MODE_DCT4X8, MODE_AFV, MODE_DCT, MODE_RAW = range(1, 8)

# AFV frequencies and their range (quant_weights.rs:989-1012), f32 constants
AFV_FREQS = np.array(F32([0xBAD, 0xBAD, 0.8517778890324296, 5.37778436506804, 0xBAD, 0xBAD, 4.734747904497923,
                          5.449245381693219, 1.6598270267479331, 4.0, 7.275749096817861, 10.423227632456525,
                          2.662932286148962, 7.630657783650829, 8.962388608184032, 12.97166202570235]), np.float64)
AFV_LO = float(F32(0.8517778890324296))
AFV_HI = float(F32(F32(12.97166202570235) - F32(AFV_LO)) + F32(1e-6))
SQRT2_PLUS = float(F32(np.sqrt(2.0)) + F32(1e-6))  # SQRT_2 + 1e-6 (get_quant_weights, :1156)


class Refused(Exception):
    """The reference returns an error for this encoding (the name of its Error variant)."""


def num_entries(idx):
    return 64 * REQUIRED_SIZE_X[idx] * REQUIRED_SIZE_Y[idx]


def f16(bits):
    """f16 bit patterns -> float64, exactly (subnormals, inf and NaN included)."""
    return np.asarray(bits, np.int64).astype(np.uint16).view(np.float16).astype(np.float64)


def f16_bits(values):
    """Nearest f16 bit patterns of float values (a helper for writing encodings)."""
    return np.asarray(values, np.float64).astype(np.float16).view(np.uint16).astype(np.int64)


# ---------------------------------------------------------------------------------------------------------------------
# Library encodings (quant_weights.rs:347-880) from quant_params.inc
# ---------------------------------------------------------------------------------------------------------------------
def _read_params():
    """{name: (3, N) float64} of every table in quant_params.inc; an entry may be a product of literals."""
    text = open(os.path.join(ROOT, "jxl_rs_b200", "csrc", "host", "quant_params.inc")).read()
    body = "\n".join(line.split("//")[0] for line in text.splitlines())
    out = {}
    for decl in body.split(";"):
        if "[3][" not in decl:
            continue
        name = decl.split("[3][")[0].split()[-1]
        rows = []
        for row in decl.split("=", 1)[1].split("}")[:3]:
            vals = []
            for entry in row.replace("{", "").split(","):
                if not entry.strip():
                    continue
                v = F32(1.0)
                for lit in entry.split("*"):
                    v = F32(v * F32(float(lit.strip().rstrip("f"))))
                vals.append(float(v))
            rows.append(vals)
        out[name] = np.array(rows, np.float64)
    return out


_PARAMS = None


def library_encoding(idx):
    """The library default of table idx (get_library_encoding, quant_weights.rs:858-880), values as floats."""
    global _PARAMS
    if _PARAMS is None:
        _PARAMS = _read_params()
    p = _PARAMS
    dct_names = {0: "k_dct_0", 4: "k_dct16x16_0", 5: "k_dct32x32_0", 6: "k_dct8x16_0", 7: "k_dct8x32_0",
                 8: "k_dct16x32_0", 11: "k_dct64x64_0", 12: "k_dct32x64_0", 13: "k_dct128x128_0",
                 14: "k_dct64x128_0", 15: "k_dct256x256_0", 16: "k_dct128x256_0"}
    if idx in dct_names:
        return {"library": True, "mode": MODE_DCT, "dct": p[dct_names[idx]]}
    if idx == 1:
        return {"library": True, "mode": MODE_IDENTITY, "w": p["k_id_0"]}
    if idx == 2:
        return {"library": True, "mode": MODE_DCT2, "w": p["k_dct2x2_0"]}
    if idx == 3:
        return {"library": True, "mode": MODE_DCT4, "w": p["k_dct4x4_1"], "dct": p["k_dct4x4_0"]}
    if idx == 9:
        return {"library": True, "mode": MODE_DCT4X8, "w": np.ones(3), "dct": p["k_dct4x8_0"]}
    if idx == 10:
        return {"library": True, "mode": MODE_AFV, "w": p["k_afv0_0"], "dct": p["k_dct4x8_0"], "dct4": p["k_dct4x4_0"]}
    raise ValueError(f"table index {idx}")


# ---------------------------------------------------------------------------------------------------------------------
# Reading an encoding (QuantEncoding::decode, quant_weights.rs:117-255; DctQuantWeightParams::decode, :58-71)
# ---------------------------------------------------------------------------------------------------------------------
def _dct_params(rows):
    p = f16(rows).reshape(3, -1).copy()
    if not 1 <= p.shape[1] <= 16:
        raise ValueError("num_bands must be 1..16")
    for c in range(3):
        if p[c, 0] < ALMOST_ZERO:
            raise Refused("HfQuantFactorTooSmall")
        p[c, 0] *= 64.0
    return p


def _checked(w):
    if (np.abs(w) < ALMOST_ZERO).any():
        raise Refused("HfQuantFactorTooSmall")
    return w


def decode(enc, idx):
    """A custom encoding (f16 bit patterns) as the reader leaves it: float values, x 64 where the reference scales."""
    mode = int(enc["mode"])
    if mode in (1, 2, 3, 4, 5) and REQUIRED_SIZE_X[idx] * REQUIRED_SIZE_Y[idx] != 1:
        raise Refused("InvalidQuantEncoding")
    v = {"mode": mode}
    if mode in (MODE_IDENTITY, MODE_DCT2):
        v["w"] = _checked(f16(enc["w"]).reshape(3, -1)) * 64.0
    elif mode == MODE_DCT4:
        v["w"] = _checked(f16(enc["w"]).reshape(3, 2))
        v["dct"] = _dct_params(enc["dct"])
    elif mode == MODE_DCT4X8:
        v["w"] = _checked(f16(enc["w"]).reshape(3))
        v["dct"] = _dct_params(enc["dct"])
    elif mode == MODE_AFV:
        w = f16(enc["w"]).reshape(3, 9).copy()
        w[:, :6] *= 64.0
        v["w"], v["dct"], v["dct4"] = w, _dct_params(enc["dct"]), _dct_params(enc["dct4"])
    elif mode == MODE_DCT:
        v["dct"] = _dct_params(enc["dct"])
    elif mode == MODE_RAW:
        v["den"] = float(f16(enc["den"]))
        if v["den"] < ALMOST_ZERO:
            raise Refused("InvalidRawQuantTable")
        raw = np.asarray(enc["raw"], np.int64).reshape(3, -1)
        if raw.shape[1] != num_entries(idx):
            raise ValueError("RAW table of the wrong size")
        if (raw <= 0).any():
            raise Refused("InvalidRawQuantTable")
        v["raw"] = raw
    else:
        raise ValueError(f"mode {mode}")
    return v


# ---------------------------------------------------------------------------------------------------------------------
# Computing the table (compute_table, quant_weights.rs:894-1079; get_quant_weights and helpers, :1138-1199)
# ---------------------------------------------------------------------------------------------------------------------
def mult(v):
    return 1.0 + v if v > 0 else 1.0 / (1.0 - v)


def _bands(first, params):
    """bands[0] = first, bands[i] = bands[i - 1] * mult(params[i]); each must stay >= ALMOST_ZERO. One zero band
    follows the last (bands[num_bands] = 0 in interpolate_vec's array)."""
    b = np.zeros(len(params) + 1)
    b[0] = first
    if b[0] < ALMOST_ZERO:  # NaN passes, as in the reference, and fails the final range check
        raise Refused("InvalidDistanceBand")
    for i in range(1, len(params)):
        b[i] = b[i - 1] * mult(params[i])
        if b[i] < ALMOST_ZERO:
            raise Refused("InvalidDistanceBand")
    return b


def _interp(bands, pos):
    """a (b / a)^frac with a = bands[floor(pos)], b = the next band; returns (weight, relative magnitude)."""
    i = np.floor(pos).astype(np.int64)
    frac = pos - i
    a, b = bands[i], bands[i + 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        w = (b / a) ** frac * a
        rel = 1.0 + i + np.where((a > 0) & (b > 0), np.abs(np.log(b / a)) * pos, 0.0)
    return w, rel


def get_quant_weights(rows, cols, p):
    """(3, rows * cols) weights and relative magnitudes (quant_weights.rs:1138-1175)."""
    nb = p.shape[1]
    w = np.zeros((3, rows * cols))
    rel = np.ones((3, rows * cols))
    scale = (nb - 1) / SQRT2_PLUS
    dy = np.arange(rows)[:, None] * (scale / (rows - 1))
    dx = np.arange(cols)[None, :] * (scale / (cols - 1))
    dist = np.sqrt(dx * dx + dy * dy).reshape(-1)
    for c in range(3):
        bands = _bands(p[c, 0], p[c, :nb])
        if nb == 1:
            w[c] = bands[0]
        else:
            w[c], rel[c] = _interp(bands, dist)
    return w, rel


def _afv_weights(v):
    w = np.zeros((3, 64))
    rel = np.ones((3, 64))
    w48, r48 = get_quant_weights(4, 8, v["dct"])
    w44, r44 = get_quant_weights(4, 4, v["dct4"])
    aw = v["w"]
    for c in range(3):
        bands = _bands(aw[c, 5], aw[c, 5:9])

        def put(x, y, val, r=1.0):
            w[c, y * 8 + x] = val
            rel[c, y * 8 + x] = r
        w[c, 0] = 1.0
        put(0, 1, aw[c, 0])
        put(1, 0, aw[c, 1])
        put(0, 2, aw[c, 2])
        put(2, 0, aw[c, 3])
        put(2, 2, aw[c, 4])
        for y in range(4):
            for x in range(4):
                if x < 2 and y < 2:
                    continue
                pos = (AFV_FREQS[y * 4 + x] - AFV_LO) * 3.0 / AFV_HI  # interpolate, :1186-1192
                val, r = _interp(bands, np.array(pos))
                put(2 * x, 2 * y, float(val), float(r))
        for y in range(4):
            for x in range(8):
                if x or y:
                    w[c, (2 * y + 1) * 8 + x] = w48[c, y * 8 + x]
                    rel[c, (2 * y + 1) * 8 + x] = r48[c, y * 8 + x]
        for y in range(4):
            for x in range(4):
                if x or y:
                    w[c, 2 * y * 8 + 2 * x + 1] = w44[c, y * 4 + x]
                    rel[c, 2 * y * 8 + 2 * x + 1] = r44[c, y * 4 + x]
    return w, rel


def raw_weights(v, idx):
    """RAW: weight i = 1 / (den * qtable[i]), the entries in the order decode_quant_table reads them."""
    return 1.0 / (v["den"] * v["raw"].astype(np.float64))


def weights(v, idx):
    """(3, num) weights before the final inversion, and their relative magnitudes."""
    mode, n = v["mode"], num_entries(idx)
    rel = np.ones((3, n))
    if mode == MODE_IDENTITY:
        w = np.repeat(v["w"][:, :1], 64, axis=1)
        w[:, 1] = w[:, 8] = v["w"][:, 1]
        w[:, 9] = v["w"][:, 2]
    elif mode == MODE_DCT2:
        xw = v["w"]
        w = np.zeros((3, 8, 8))
        w[:, 0, 0] = 0xBAD
        w[:, 0, 1] = w[:, 1, 0] = xw[:, 0]
        w[:, 1, 1] = xw[:, 1]
        w[:, 0:2, 2:4] = w[:, 2:4, 0:2] = xw[:, 2, None, None]
        w[:, 2:4, 2:4] = xw[:, 3, None, None]
        w[:, 0:4, 4:8] = w[:, 4:8, 0:4] = xw[:, 4, None, None]
        w[:, 4:8, 4:8] = xw[:, 5, None, None]
        w = w.reshape(3, 64)
    elif mode == MODE_DCT4:
        w44, r44 = get_quant_weights(4, 4, v["dct"])
        up = np.array([(y // 2) * 4 + x // 2 for y in range(8) for x in range(8)])
        w, rel = w44[:, up].copy(), r44[:, up].copy()
        w[:, 1] /= v["w"][:, 0]
        w[:, 8] /= v["w"][:, 0]
        w[:, 9] /= v["w"][:, 1]
        rel[:, [1, 8, 9]] += 1.0
    elif mode == MODE_DCT4X8:
        w48, r48 = get_quant_weights(4, 8, v["dct"])
        up = np.array([(y // 2) * 8 + x for y in range(8) for x in range(8)])
        w, rel = w48[:, up].copy(), r48[:, up].copy()
        w[:, 8] /= v["w"]
        rel[:, 8] += 1.0
    elif mode == MODE_DCT:
        w, rel = get_quant_weights(8 * REQUIRED_SIZE_X[idx], 8 * REQUIRED_SIZE_Y[idx], v["dct"])
    elif mode == MODE_RAW:
        w = raw_weights(v, idx)
    elif mode == MODE_AFV:
        w, rel = _afv_weights(v)
    else:
        raise ValueError(f"mode {mode}")
    return w, rel


def compute_table(enc, idx):
    """(table, M), each (3, 64 REQUIRED_SIZE_X REQUIRED_SIZE_Y) float64: 1 / weight after the reference's range check
    (every weight in [ALMOST_ZERO, 1 / ALMOST_ZERO], else InvalidQuantizationTableWeight). Raises Refused."""
    v = enc if enc.get("library") else decode(enc, idx)
    w, rel = weights(v, idx)
    with np.errstate(invalid="ignore"):
        ok = (w >= ALMOST_ZERO) & (w <= MAX_WEIGHT)
    if not ok.all():
        raise Refused("InvalidQuantizationTableWeight")
    table = 1.0 / w
    return table, table * rel


def table_for_transform(t, encodings=None):
    """(table, M) of transform type t: the custom encoding of its table index from `encodings` (17 entries, None =
    library), else the library default."""
    idx = TABLE_OF_TRANSFORM[t]
    enc = encodings[idx] if encodings is not None and encodings[idx] is not None else library_encoding(idx)
    return compute_table(enc, idx)


def check_table(got, ref, mag, what=""):
    """|got - ref| <= K_Q 2^-24 M for every entry; returns the largest err / (2^-24 M)."""
    got = np.asarray(got, np.float64).reshape(ref.shape)
    err = np.abs(got - ref)
    ratio = float((err / (EPS * mag)).max())
    bad = ~(err <= K_Q * EPS * mag)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} table entries outside K_q={K_Q}; largest "
                           f"err/(2^-24 M) = {ratio:.3g}; first at {np.argwhere(bad)[0].tolist()}")
    return ratio


# ---------------------------------------------------------------------------------------------------------------------
# Random valid encodings
# ---------------------------------------------------------------------------------------------------------------------
def permitted_modes(idx):
    return [1, 2, 3, 4, 5, 6, 7] if REQUIRED_SIZE_X[idx] * REQUIRED_SIZE_Y[idx] == 1 else [6, 7]


def random_encoding(rng, idx, mode, num_bands=None):
    """A random encoding the reference accepts, chosen so that no weight comes near the range limits: first bands
    and direct weights 64 x [0.5, 200], mult parameters in [-1.5, 0.5] (a factor 0.4 to 1.5 per band), DCT4 / DCT4X8
    divisors in [0.5, 2], RAW entries 1..1000 with den in [2^-16, 2^-12] (table entries 1.5e-5 to 0.24,
    about the range of the library's)."""
    def f(lo, hi, shape):
        return f16_bits(rng.uniform(lo, hi, shape))

    def dct(nb=None):
        nb = nb or int(rng.integers(1, 17))
        return np.concatenate([f(0.5, 200.0, (3, 1)), f(-1.5, 0.5, (3, nb - 1))], axis=1)
    if mode == MODE_IDENTITY:
        return {"mode": mode, "w": f(0.5, 200.0, (3, 3))}
    if mode == MODE_DCT2:
        return {"mode": mode, "w": f(0.5, 200.0, (3, 6))}
    if mode == MODE_DCT4:
        return {"mode": mode, "w": f(0.5, 2.0, (3, 2)), "dct": dct(num_bands)}
    if mode == MODE_DCT4X8:
        return {"mode": mode, "w": f(0.5, 2.0, 3), "dct": dct(num_bands)}
    if mode == MODE_AFV:
        return {"mode": mode, "w": np.concatenate([f(0.5, 200.0, (3, 6)), f(-1.5, 0.5, (3, 3))], axis=1),
                "dct": dct(num_bands), "dct4": dct()}
    if mode == MODE_DCT:
        return {"mode": mode, "dct": dct(num_bands)}
    if mode == MODE_RAW:
        h, w = 8 * REQUIRED_SIZE_Y[idx], 8 * REQUIRED_SIZE_X[idx]
        return {"mode": mode, "den": int(f(2.0 ** -16, 2.0 ** -12, ())), "raw": rng.integers(1, 1001, (3, h, w))}
    raise ValueError(f"mode {mode}")


def profile4_encodings(seed, modes=None):
    """Custom encodings for all 17 tables: RAW at 0, 6 (non-square) and 11 (square), the special 8x8 modes at 1, 2, 3,
    9 and 10, DCT elsewhere; `modes` overrides."""
    rng = np.random.default_rng(seed)
    m = {0: MODE_RAW, 1: MODE_IDENTITY, 2: MODE_DCT2, 3: MODE_DCT4, 6: MODE_RAW, 9: MODE_DCT4X8,
         10: MODE_AFV, 11: MODE_RAW}
    m.update(modes or {})
    return [None if m.get(i, MODE_DCT) is None else random_encoding(rng, i, m.get(i, MODE_DCT))
            for i in range(17)]


def tables_used(fr):
    """The table indices the varblocks of a frame read (from its transform map)."""
    tm = fr.transform_map
    return {TABLE_OF_TRANSFORM[int(t) & 127] for t in np.unique(tm[tm >= 128])}


def assert_custom_tables_used(fr, encodings, what):
    unused = [i for i, e in enumerate(encodings) if e is not None and i not in tables_used(fr)]
    assert not unused, f"{what}: custom tables {unused} are read by no varblock"
