"""Output colour of XYB images (SURVEY §8 a15/a16): the host front-end's OutputColorInfo derivation and the oracle's
from_linear curves, checked against independent float64 numpy restatements written from the reference
(render/stages/xyb.rs:65-140, api/color.rs:124-275, color/tf.rs). The reference's own tests hold its rational
approximations to the exact curves within 8e-7 (PQ, tf.rs:626-639), 1e-6 (sRGB / BT.709, tf.rs:600-624) and the
fast_powf error 3e-5 (util/fast_math.rs:151); the same bars are used here. No GPU."""
import ctypes as C

import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests.f64_pipeline import bt709_exact, gamma_exact, hlg_exact, pq_exact

OPSIN_INV = np.array([[11.031566901960783, -9.866943921568629, -0.16462299647058826],
                      [-3.254147380392157, 4.418770392156863, -0.16462299647058826],
                      [-3.6588512862745097, 2.7129230470588235, 1.9459282392156863]])
BRADFORD = np.array([[0.8951, 0.2664, -0.1614], [-0.7502, 1.7135, 0.0367], [0.0389, -0.0685, 1.0296]])
BRADFORD_INV = np.array([[0.9869929, -0.1470543, 0.1599627], [0.4323053, 0.5183603, 0.0492912], [-0.0085287, 0.0400428, 0.9684867]])
SRGB = [(0.6399987, 0.33001015), (0.3000038, 0.60000336), (0.15000205, 0.059997204)]
BT2100 = [(0.708, 0.292), (0.170, 0.797), (0.131, 0.046)]
P3 = [(0.680, 0.320), (0.265, 0.690), (0.150, 0.060)]
D65, DCI, E = (0.3127, 0.3290), (0.314, 0.351), (1 / 3, 1 / 3)


def f32(v):
    return float(np.float32(v))


def primaries_to_xyz(prim, w):  # api/color.rs:124-190
    prim = [(f32(x), f32(y)) for x, y in prim]
    wx, wy = f32(w[0]), f32(w[1])
    p = np.array([[x for x, _ in prim], [y for _, y in prim], [1 - x - y for x, y in prim]])
    s = np.linalg.solve(p, np.array([wx / wy, 1.0, (1 - wx - wy) / wy]))
    return p @ np.diag(s)


def adapt_to_d50(w):  # api/color.rs:193-252
    wx, wy = f32(w[0]), f32(w[1])
    src = BRADFORD @ np.array([wx / wy, 1.0, (1 - wx - wy) / wy])
    dst = BRADFORD @ np.array([0.96422, 1.0, 0.82521])
    return BRADFORD_INV @ np.diag(dst / src) @ BRADFORD


def expected_matrix(prim, w):  # render/stages/xyb.rs:92-107
    srgb_to_d50 = adapt_to_d50(D65) @ primaries_to_xyz(SRGB, D65)
    orig_to_xyz = primaries_to_xyz(prim, w)
    orig_to_d50 = adapt_to_d50(w) @ orig_to_xyz
    return np.linalg.inv(orig_to_d50) @ srgb_to_d50 @ np.float32(OPSIN_INV).astype(np.float64), orig_to_xyz[1]


def output_colour(cs=0, wp=1, wxy=None, pr=1, pxy=None, have_gamma=0, gamma=0, tf=13):
    from tests import oracle_binding as ob
    lib = ob.load()
    out = (C.c_float * 14)()
    w = (C.c_int32 * 2)(*(wxy or (0, 0)))
    p = (C.c_int32 * 6)(*(pxy or (0,) * 6))
    r = lib.jxo_t_output_colour(cs, wp, w, pr, p, have_gamma, gamma, tf, out)
    v = np.array(list(out), np.float64)
    return r, v[:9].reshape(3, 3), v[9:12], int(v[12]), v[13]


@pytest.mark.parametrize("name,pr,prim,wp,white", [("P3-D65", 11, P3, 1, D65), ("BT2100-D65", 9, BT2100, 1, D65),
                                                   ("sRGB-DCI", 1, SRGB, 11, DCI), ("P3-E", 11, P3, 10, E)])
def test_matrix_retargeting(name, pr, prim, wp, white):
    r, m, lum, tf, _ = output_colour(wp=wp, pr=pr)
    assert r == 0 and tf == abi_tf("SRGB")
    want, want_lum = expected_matrix(prim, white)
    assert np.allclose(m, want, rtol=2e-6, atol=2e-6), f"{name}: {np.abs(m - want).max()}"
    assert np.allclose(lum, want_lum, rtol=1e-6)


def test_custom_chromaticities_equal_named_ones():
    """Custom xy values in 1e-6 units (color_encoding.rs:91-106) of P3 / DCI give the matrix of the named enums."""
    pxy = [int(round(v * 1e6)) for xy in P3 for v in xy]
    wxy = [int(round(v * 1e6)) for v in DCI]
    r0, m0, l0, _, _ = output_colour(wp=11, pr=11)
    r1, m1, l1, _, _ = output_colour(wp=2, wxy=wxy, pr=2, pxy=pxy)
    assert r0 == 0 and r1 == 0
    assert np.allclose(m0, m1, rtol=1e-5, atol=1e-5) and np.allclose(l0, l1, rtol=1e-5)


def test_srgb_d65_keeps_the_opsin_matrix_and_grey_folds_luminances():
    r, m, lum, tf, _ = output_colour()
    assert r == 0 and np.array_equal(m, np.float32(OPSIN_INV).astype(np.float64)) and tf == 1
    r, m, _, _, _ = output_colour(cs=1)  # grey: every row = luminances . matrix (xyb.rs:110-118)
    row = np.float32([0.2126, 0.7152, 0.0722]).astype(np.float64) @ np.float32(OPSIN_INV).astype(np.float64)
    assert r == 0 and np.allclose(m, np.stack([row] * 3), rtol=1e-6)


def abi_tf(name):
    return {"LINEAR": 0, "SRGB": 1, "GAMMA": 2, "BT709": 3, "PQ": 4, "HLG": 5}[name]


def test_transfer_function_mapping_and_refusals():
    assert output_colour(tf=8)[3] == abi_tf("LINEAR")
    assert output_colour(tf=1)[3] == abi_tf("BT709")
    assert output_colour(tf=16)[3] == abi_tf("PQ")
    assert output_colour(tf=18)[3] == abi_tf("HLG")
    r, _, _, tf, g = output_colour(tf=17)  # DCI = gamma 1 / 2.6 (xyb.rs:130)
    assert r == 0 and tf == abi_tf("GAMMA") and abs(g - 1 / 2.6) < 1e-7
    r, _, _, tf, g = output_colour(have_gamma=1, gamma=4545455)
    assert r == 0 and tf == abi_tf("GAMMA") and abs(g - 0.4545455) < 1e-7
    assert output_colour(have_gamma=1, gamma=10000001)[0] != 0       # gamma > 1 (color_encoding.rs:150-157)
    assert output_colour(cs=2)[0] == -2                              # XYB colour space: no simple output profile
    assert output_colour(cs=1, wp=11)[0] == -2                       # grey, non-D65 (api/color.rs:1291-1294)
    assert output_colour(tf=2)[0] != 0                               # TransferFunction::Unknown


def from_linear(tf, rgb, gamma=1.0, it=255.0, lum=(0.2126, 0.7152, 0.0722)):
    from tests import oracle_binding as ob
    lib = ob.load()
    a = np.ascontiguousarray(rgb, np.float32).copy()
    l = (C.c_float * 3)(*lum)
    lib.jxo_from_linear.argtypes = [C.c_uint32, C.c_float, C.c_float, C.c_void_p, C.c_int, C.c_void_p]
    lib.jxo_from_linear(tf, gamma, it, l, a.shape[0], a.ctypes.data)
    return a.astype(np.float64)


def samples(seed, n=4000):
    rng = np.random.default_rng(seed)
    v = np.concatenate([rng.uniform(0, 1, (n, 3)), rng.uniform(0, 1e-3, (200, 3)), rng.uniform(-0.2, 0, (200, 3))])
    return v.astype(np.float32)


def test_gamma_bt709_curves():
    v = samples(1)
    x = v.astype(np.float64)
    got = from_linear(abi_tf("GAMMA"), v, gamma=0.45)
    want = gamma_exact(x, 0.45)
    assert np.all(np.abs(got - want) <= 1e-4 * np.maximum(np.abs(want), 1e-2))  # fast_powf: 3e-5 relative
    got = from_linear(abi_tf("BT709"), v)
    want = bt709_exact(x)
    assert np.abs(got - want).max() <= 2e-6  # tf.rs:613-624 holds the rational form to 1e-6 of the naive one


def test_pq_curve():
    for it in (10000.0, 4000.0, 255.0):
        v = samples(2)
        want = pq_exact(v.astype(np.float64), it)
        got = from_linear(abi_tf("PQ"), v, it=it)
        big = np.abs(v) >= 1e-4
        # The reference switches polynomials on the UNSCALED sample (tf.rs:269-275), so below 10000 nits the main
        # polynomial is used outside its fitted range ("Error seems to increase at intensity_target < 10000",
        # tf.rs:636): the restatement follows it, the exact curve is only close there.
        assert np.abs(got - want)[big].max() <= (2e-6 if it == 10000.0 else 5e-4)


def test_hlg_curve():
    lum = (0.2627, 0.6780, 0.0593)
    for it in (1000.0, 255.0, 4000.0):
        v = samples(3)[:4000]
        want = hlg_exact(v.astype(np.float64), it, lum)
        got = from_linear(abi_tf("HLG"), v, it=it, lum=lum)
        assert np.abs(got - want).max() <= 1e-4  # fast_powf in the OOTF (3e-5 relative), fast_log2f in the OETF (5e-7)


def test_f16_store_matches_the_reference_conversion():
    """util/float16.rs:82-141 restated with numpy: round to nearest even for normal halves, overflow to infinity, and
    TRUNCATION (not rounding) into the subnormal range (with the reference's extra halving there), zero below 2^-24 —
    the F16 output format's last step."""
    from tests import oracle_binding as ob
    lib = ob.load()
    rng = np.random.default_rng(9)
    v = np.concatenate([rng.uniform(-2, 2, 20000), rng.uniform(-1e-4, 1e-4, 20000), rng.uniform(-1e-7, 1e-7, 2000),
                        np.array([0.0, -0.0, 1.0, 65504.0, 65519.9, 65520.0, 1e6, -1e6, 2.0 ** -14, 2.0 ** -24, 2.0 ** -25,
                                  0.5 + 2.0 ** -12, 0.5 + 3 * 2.0 ** -12, 1e-45])]).astype(np.float32)
    out = np.zeros(v.shape, np.uint16)
    lib.jxo_f32_to_f16.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    lib.jxo_f32_to_f16(len(v), v.ctypes.data, out.ctypes.data)
    got = out.view(np.float16).astype(np.float64)
    a = np.abs(v.astype(np.float64))
    with np.errstate(over="ignore"):
        rne = v.astype(np.float16).astype(np.float64)  # IEEE round to nearest even (numpy)
    normal = a >= 2.0 ** -14
    assert np.array_equal(got[normal], rne[normal])
    sub = (a < 2.0 ** -14) & (a >= 2.0 ** -24)
    # float16.rs:104-108 shifts the 24-bit significand by (-14 - e) + 14 bits, one more than the value needs: inputs in the
    # subnormal range come out truncated AND halved (2^-15 -> 2^-16). Reproduced as is - identical output is the contract.
    want = np.sign(v[sub]) * np.floor(a[sub] * 2.0 ** 23) * 2.0 ** -24
    assert np.array_equal(got[sub], want)
    tiny = a < 2.0 ** -24
    assert np.all(got[tiny] == 0.0)
    assert np.array_equal(np.signbit(got), np.signbit(v.astype(np.float64)))
