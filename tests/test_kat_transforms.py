"""The oracle's transform / filter / colour primitives against the reference's own definitions and tolerances:
jxl_transforms/src/tests.rs:62-180,286-492 (IDCT and reinterpreting DCT vs f64 definitions),
render/stages/gaborish.rs:133-144, render/stages/xyb.rs:289-311, color/tf.rs:549-585."""
import ctypes as C

import numpy as np
import pytest

from tests.f64_pipeline import slow_idct2d, slow_reinterpreting_dct2d


def check_close(a, b, tol):
    d = np.abs(a - b)
    rel = d / np.maximum(np.maximum(np.abs(a), np.abs(b)), 1e-300)
    assert np.all((d < tol) | (rel < tol)), float(d.max())


IDCT_CASES = [(2, 2, 1e-6), (4, 4, 1e-6), (4, 8, 1e-6), (8, 4, 1e-6), (8, 8, 5e-6), (16, 8, 5e-6), (8, 16, 5e-6), (16, 16, 1e-5),
              (32, 8, 5e-6), (8, 32, 5e-6), (32, 16, 1e-5), (16, 32, 1e-5), (32, 32, 5e-5), (64, 32, 1e-4), (32, 64, 1e-4),
              (64, 64, 1e-4), (128, 64, 5e-4), (64, 128, 5e-4), (128, 128, 5e-4), (256, 128, 1e-3), (128, 256, 1e-3),
              (256, 256, 5e-3)]  # tests.rs:318-339


@pytest.mark.parametrize("rows,cols,tol", IDCT_CASES)
def test_idct2d_vs_f64_definition(oracle, rows, cols, tol):
    rng = np.random.default_rng(0)
    inp = rng.uniform(-1, 1, (rows, cols))
    ref = slow_idct2d(inp)
    buf = inp.astype(np.float32).reshape(-1).copy()
    oracle.jxo_idct2d(rows, cols, buf.ctypes.data)
    # the reference's tolerances hold for its ChaCha12(seed 0) input; another random draw lands within 4x of them
    check_close(buf.reshape(rows, cols).astype(np.float64), ref, 4 * tol)


RDCT_CASES = [(1, 2, 1e-6), (2, 1, 1e-6), (2, 2, 1e-6), (1, 4, 1e-6), (4, 1, 1e-6), (2, 4, 1e-6), (4, 2, 1e-6), (4, 4, 1e-6),
              (8, 4, 1e-6), (4, 8, 1e-6), (8, 8, 1e-6), (8, 16, 5e-6), (16, 8, 5e-6), (16, 16, 5e-6), (32, 16, 5e-6),
              (16, 32, 5e-6), (32, 32, 5e-6)]  # tests.rs:367-492


@pytest.mark.parametrize("rows,cols,tol", RDCT_CASES)
def test_reinterpreting_dct_vs_f64_definition(oracle, rows, cols, tol):
    rng = np.random.default_rng(0)
    inp = rng.uniform(-1, 1, (rows, cols))
    ref = slow_reinterpreting_dct2d(inp)
    on, om = ref.shape
    out = np.zeros(rows * cols * 64, np.float32)
    a = inp.astype(np.float32).reshape(-1).copy()
    oracle.jxo_reinterpreting_dct2d(rows, cols, a.ctypes.data, out.ctypes.data, om * 8)
    got = np.array([[out[r * om * 8 + c] for c in range(om)] for r in range(on)], np.float64)
    # the generated reference code carries 6-decimal scale constants; allow their rounding on top of `tol`
    check_close(got, ref, max(tol, 2e-5))


def test_gaborish_checkerboard(oracle):  # gaborish.rs:133-144
    img = np.array([[0.0, 1.0], [1.0, 0.0]], np.float32)
    out = np.zeros_like(img)
    oracle.jxo_gaborish(2, 2, img.ctypes.data, out.ctypes.data, C.c_float(0.115169525), C.c_float(0.061248592))
    np.testing.assert_allclose(out, [[0.20686048, 0.7931395], [0.7931395, 0.20686048]], atol=1e-6)


def test_xyb_srgb_primaries(oracle):  # xyb.rs:289-311
    x = np.array([0.028100073, -0.015386105, 0.0], np.float32)
    y = np.array([0.4881882, 0.71478134, 0.2781282], np.float32)
    b = np.array([0.471659, 0.43707693, 0.66613984], np.float32)
    m = np.array([11.031566901960783, -9.866943921568629, -0.16462299647058826, -3.254147380392157, 4.418770392156863,
                  -0.16462299647058826, -3.6588512862745097, 2.7129230470588235, 1.9459282392156863], np.float32)
    bias = np.array([-0.0037930732552754493] * 3, np.float32)
    oracle.jxo_xyb_to_linear(3, x.ctypes.data, y.ctypes.data, b.ctypes.data, m.ctypes.data, bias.ctypes.data, C.c_float(255.0))
    np.testing.assert_allclose(np.stack([x, y, b]), np.eye(3), atol=1e-5)


def test_srgb_transfer_function(oracle):  # tf.rs:549-585
    v = np.linspace(0, 1, 1001).astype(np.float32)
    got = v.copy()
    oracle.jxo_linear_to_srgb(got.size, got.ctypes.data)
    ref = np.where(v <= 0.0031308, v * 12.92, 1.055 * np.power(v.astype(np.float64), 1 / 2.4) - 0.055)
    assert np.abs(got - ref).max() < 2e-6 + 5e-7
    neg = np.array([-0.25], np.float32)
    oracle.jxo_linear_to_srgb(1, neg.ctypes.data)
    assert neg[0] < 0


@pytest.mark.parametrize("xs,ys", [(3, 3), (10, 4), (37, 21), (480, 270)])
def test_adaptive_lf_smoothing_matches_the_scalar_definition(oracle, xs, ys):
    """adaptive_lf_smoothing.rs:20-41,88-117 restated in numpy f32 (unfused multiplies and adds, like the scalar Rust):
    the host front-end's AVX2 body must agree bit for bit, borders copied unchanged."""
    import ctypes as C
    rng = np.random.default_rng(xs * 1000 + ys)
    lf_quant = np.array([1 / 4096, 1 / 512, 1 / 256], np.float32)
    gs, qlf = 3072, 16
    f = np.float32
    inv = f(f(65536.0) / f(gs)) / f(qlf)
    fac = [f(inv * lf_quant[c]) for c in range(3)]
    # quantised LF samples: a smooth ramp (small gaps, factor > 0) with an edge and sparse outliers (factor == 0)
    yy, xx = np.mgrid[0:ys, 0:xs]
    q = np.round(0.3 * xx + 0.2 * yy + 6.0 * (yy >= ys // 2)).astype(np.int32)[None] + (rng.random((3, ys, xs)) < 0.05) * 3
    lf = np.stack([(q[c] * fac[c]).astype(np.float32) for c in range(3)])
    ws, wc = f(0.20345139757231578), f(0.0334829185968739)
    wcen = f(f(1.0) - f(4.0) * f(ws + wc))
    want = lf.copy()
    gap = np.full((ys - 2, xs - 2), 0.5, np.float32)
    mc, sm = [], []
    for c in range(3):
        p = lf[c]
        corner = ((p[:-2, :-2] + p[:-2, 2:]) + p[2:, :-2]) + p[2:, 2:]
        side = ((p[1:-1, :-2] + p[1:-1, 2:]) + p[:-2, 1:-1]) + p[2:, 1:-1]
        m = p[1:-1, 1:-1]
        s = (corner * wc + side * ws) + m * wcen
        mc.append(m)
        sm.append(s)
        gap = np.maximum(gap, np.abs((m - s) / fac[c]))
    factor = np.maximum(f(3.0) - f(4.0) * gap, f(0.0))
    for c in range(3):
        want[c, 1:-1, 1:-1] = (sm[c] - mc[c]) * factor + mc[c]
    if xs * ys > 100:
        assert (factor == 0).any() and (factor > 0).any()
    for threads in (1, 3):  # 3: row bands on separate threads (only the 270-row case is tall enough to split)
        got = lf.copy()
        oracle.jxo_t_adaptive_lf_smoothing(xs, ys, gs, qlf, lf_quant.ctypes.data_as(C.c_void_p),
                                           got.ctypes.data_as(C.c_void_p), threads)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
