"""Float stages of the VarDCT path pinned independently of the oracle's C++ (SURVEY §8 a9, a10-LF, a13, a14): float64 numpy
restatements written from the reference sources — render/stages/epf/{epf0,epf1,epf2,common}.rs, features/epf.rs:35-86,
frame/group.rs:85-177 (adjust_quant_bias, dequant_lane, chroma from luma) and frame/modular/mod.rs:837-929 (dequant_lf)
— against the oracle on random inputs with a random sigma image, the set-up of the reference's own EPF tests
(render/stages/epf/test.rs:15-49, which only compare SIMD levels with each other). The reference holds no vector for
these stages, so this is the strongest pin available without a Rust toolchain: two implementations written separately
from the same text, one in f32 with the reference's operation order, one in f64 as plain array arithmetic.
Tolerance 1e-5 (relative to the value range of the planes, which are O(1)). No GPU."""
import ctypes as C

import numpy as np
import pytest

from tests.f64_pipeline import MIN_SIGMA, epf_stage_f64, sigma_image_f64
from tests.f64_prefix import dequant_lf_f64


def _lib():
    from tests import oracle_binding as ob
    lib = ob.load()
    f, vp, u32, i32 = C.c_float, C.c_void_p, C.c_uint32, C.c_int32
    lib.jxo_dequant_block.argtypes = [u32, vp, vp, vp, vp, f, f, f, f, f, vp, vp]
    lib.jxo_sigma_image.argtypes = [u32, u32, u32, vp, vp, f, vp, vp]
    lib.jxo_epf_stage.argtypes = [C.c_int, u32, u32, vp, vp, vp, vp, f, f, f, C.c_int]
    lib.jxo_t_dequant_lf.argtypes = [u32, u32, vp, u32, u32, vp, u32, f, f, i32, i32, u32, vp, vp, vp, vp]
    return lib


# ---------------------------------------------------------------------------------------------------------------------
# EPF
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stage", [0, 1, 2])
@pytest.mark.parametrize("shape", [(96, 64), (61, 43), (8, 8), (5, 3)])
def test_epf_stage_against_f64_restatement(stage, shape):
    lib = _lib()
    w, h = shape
    rng = np.random.default_rng(1000 * stage + w)
    # smooth picture + noise + an edge, X / Y / B value ranges of a real XYB image
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([0.01 * np.sin(xx / 7.0), 0.4 + 0.2 * np.cos(yy / 9.0), 0.3 + 0.1 * np.sin((xx + yy) / 11.0)])
    img = (base + rng.normal(0, [[[0.002]], [[0.02]], [[0.02]]], (3, h, w)) + (xx > w // 2) * np.array([0.005, 0.1, 0.08])[:, None, None])
    img = img.astype(np.float32)
    xb, yb = (w + 7) // 8, (h + 7) // 8
    raw_quant = rng.integers(1, 40, (yb, xb)).astype(np.int32)
    sharp = rng.integers(0, 8, (yb, xb)).astype(np.uint8)
    lut = (np.arange(8) / 7.0).astype(np.float32)
    sig32 = np.zeros((yb, xb), np.float32)
    lib.jxo_sigma_image(xb, yb, 4000, raw_quant.ctypes.data, sharp.ctypes.data, 0.46, lut.ctypes.data, sig32.ctypes.data)
    want_sig = sigma_image_f64(4000, raw_quant, sharp, np.float32(0.46), lut)
    assert np.allclose(sig32, want_sig, rtol=2e-6)
    if xb * yb >= 12:
        assert (sig32 < MIN_SIGMA).any() and (sig32 >= MIN_SIGMA).any()  # both branches of the pass-through
    cs = np.array([40.0, 5.0, 3.5], np.float32)
    out = np.zeros_like(img)
    lib.jxo_epf_stage(stage, w, h, img.ctypes.data, out.ctypes.data, sig32.ctypes.data, cs.ctypes.data, 0.9, 6.5, 2.0 / 3.0, 2)
    scale = {0: np.float32(0.9), 1: 1.0, 2: np.float32(6.5)}[stage]
    want = epf_stage_f64(stage, img.astype(np.float64), sig32.astype(np.float64), cs, float(scale), float(np.float32(2.0 / 3.0)))
    assert np.abs(out - want).max() <= 1e-5, np.abs(out - want).max()
    if (sig32 >= MIN_SIGMA).any():
        assert np.abs(out - img).max() > 1e-4  # the filter did something


# ---------------------------------------------------------------------------------------------------------------------
# HF dequantisation + chroma from luma
# ---------------------------------------------------------------------------------------------------------------------
def test_dequant_block_against_f64_restatement():
    lib = _lib()
    rng = np.random.default_rng(7)
    for n in (64, 256, 1024):
        q = rng.integers(-6, 7, (3, n)).astype(np.int32)
        q[:, rng.random(n) < 0.5] = 0
        q[1, :8] = [0, 1, -1, 2, -2, 3, -40, 1000]
        mat = rng.uniform(1e-3, 2.0, (3, n)).astype(np.float32)
        bias = np.array([0.94534993, 0.92994550, 0.95006490, 0.145], np.float32)
        inv_global_scale, raw_quant = np.float32(65536.0 / 4587), 5
        sy = np.float32(inv_global_scale / np.float32(raw_quant))
        sx, sb = np.float32(sy * np.float32(0.8)), np.float32(sy * np.float32(1.0))
        x_cc, b_cc = np.float32(0.0 + 3 / 84.0), np.float32(1.0 - 5 / 84.0)
        out = np.zeros((3, n), np.float32)
        lib.jxo_dequant_block(n, q[0].ctypes.data, q[1].ctypes.data, q[2].ctypes.data, mat.ctypes.data, sx, sy, sb, x_cc, b_cc,
                              bias.ctypes.data, out.ctypes.data)
        # group.rs:85-96 adjust_quant_bias, :100-133 dequant_lane, in float64
        qf, b64 = q.astype(np.float64), bias.astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            adj = np.where(np.abs(q) < 2, qf * b64[:3, None], qf - b64[3] / qf)
        d = adj * mat.astype(np.float64) * np.array([sx, sy, sb], np.float64)[:, None]
        want = np.stack([d[0] + float(x_cc) * d[1], d[1], d[2] + float(b_cc) * d[1]])
        # f32 rounding scales with the larger of the two terms of the chroma-from-luma sum
        mag = np.stack([np.abs(d[0]) + abs(float(x_cc)) * np.abs(d[1]), np.abs(d[1]), np.abs(d[2]) + abs(float(b_cc)) * np.abs(d[1])])
        assert np.all(np.abs(out - want) <= 1e-6 * mag + 1e-9), np.abs(out - want).max()


# ---------------------------------------------------------------------------------------------------------------------
# LF dequantisation (front-end) + LF context buckets
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra_precision", [0, 2])
def test_dequant_lf_against_f64_restatement(extra_precision):
    lib = _lib()
    rng = np.random.default_rng(11 + extra_precision)
    w, h = 37, 23
    q = rng.integers(-300, 300, (3, h, w)).astype(np.int32)  # coded channel order Y, X, B (modular/mod.rs:958-962)
    lf_quant = np.array([1 / 4096.0, 1 / 512.0, 1 / 256.0], np.float32)
    thr = [np.array([-20, 15], np.int32), np.array([0], np.int32), np.array([-100, 0, 120], np.int32)]  # X, Y, B thresholds
    nthr = np.array([len(t) for t in thr], np.uint32)
    tall = np.concatenate(thr).astype(np.int32)
    out = np.zeros((3, h, w), np.float32)
    qlf = np.zeros((h, w), np.uint8)
    gs, ql, cf, ytox, ytob = 4587, 16, 84, -7, 21
    lib.jxo_t_dequant_lf(w, h, q.ctypes.data, gs, ql, lf_quant.ctypes.data, extra_precision, 0.0, 1.0, ytox, ytob, cf, tall.ctypes.data,
                         nthr.ctypes.data, out.ctypes.data, qlf.ctypes.data)
    want, _ = dequant_lf_f64(q[1], q[0], q[2], gs, ql, 0.0, ytox, 1.0, ytob, cf, mul=1.0 / (1 << extra_precision),
                             lf_quant=lf_quant.astype(np.float64))
    assert np.allclose(out, want, rtol=3e-6, atol=1e-7), np.abs(out - want).max()
    # mod.rs:898-924: bucket = (bucket_x * (|thr_b| + 1) + bucket_b) * (|thr_y| + 1) + bucket_y, strict comparisons
    bx = (q[1][..., None] > thr[0]).sum(-1)
    by = (q[0][..., None] > thr[1]).sum(-1)
    bb = (q[2][..., None] > thr[2]).sum(-1)
    assert np.array_equal(qlf, ((bx * (len(thr[2]) + 1) + bb) * (len(thr[1]) + 1) + by).astype(np.uint8))


# ---- HF-metadata placement (integer; lives here with the other independent restatements of the front-end) ----
_COV_X = [1, 1, 1, 1, 2, 4, 1, 2, 1, 4, 2, 4, 1, 1, 1, 1, 1, 1, 8, 4, 8, 16, 8, 16, 32, 16, 32]
_COV_Y = [1, 1, 1, 1, 2, 4, 2, 1, 4, 1, 4, 2, 1, 1, 1, 1, 1, 1, 8, 8, 4, 16, 16, 8, 32, 32, 16]


def _place_reference(w, h, count, raw_t, raw_q):
    """modular/mod.rs:1032-1078 written out as the reference writes it: every block position in raster order; a position
    already covered is skipped; the next entry of the block list is placed there (bounds: the LF-group rect and the 32x32
    block group); covered positions are overwritten, the first one carries bit 7. covered_blocks_x/y: transform_map.rs."""
    tm = np.full((h, w), 27, np.uint8)
    rq = np.zeros((h, w), np.int32)
    num = 0
    for y in range(h):
        for x in range(w):
            if tm[y, x] != 27:
                continue
            if num >= count:
                return None
            t = int(raw_t[num])
            q = 1 + min(max(int(raw_q[num]), 0), 255)
            if not 0 <= t < 27:
                return None
            cx, cy = _COV_X[t], _COV_Y[t]
            if x + cx > min(w, (x // 32 + 1) * 32) or y + cy > min(h, (y // 32 + 1) * 32):
                return None
            num += 1
            for iy in range(cy):
                for ix in range(cx):
                    tm[y + iy, x + ix] = t | (128 if (ix == 0 and iy == 0) else 0)
                    rq[y + iy, x + ix] = q
    return tm, rq


def test_varblock_placement_against_the_reference_loop():
    """The front-end's placement loop (skips covered runs, 8x8 fast path, row pointers) against the reference's plain double
    loop, on random block lists: valid tilings with all 27 transform types, lists that run out, blocks that cross a 32x32
    group or the rect, out-of-range transform ids, quantiser values outside 0..255."""
    from tests import oracle_binding as ob
    lib = ob.load()
    lib.jxo_t_place_varblocks.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    rng = np.random.default_rng(77)
    ok = bad = 0
    for trial in range(300):
        w, h = int(rng.integers(1, 70)), int(rng.integers(1, 70))
        # build a list by simulating the placement with random transform choices that fit (or, sometimes, any choice)
        sloppy = trial % 6 == 5
        poison = trial % 9 == 8  # one out-of-range transform id somewhere in the list
        cover = np.zeros((h, w), bool)
        ts, qs = [], []
        for y in range(h):
            for x in range(w):
                if cover[y, x]:
                    continue
                cands = list(range(27))
                rng.shuffle(cands)
                t = None
                for c in cands:
                    cx, cy = _COV_X[c], _COV_Y[c]
                    if sloppy or (x + cx <= min(w, (x // 32 + 1) * 32) and y + cy <= min(h, (y // 32 + 1) * 32)
                                  and not cover[y:y + cy, x:x + cx].any()):
                        t = c
                        break
                if t is None:
                    t = 0
                cx, cy = _COV_X[t], _COV_Y[t]
                cover[y:min(h, y + cy), x:min(w, x + cx)] = True
                ts.append(t)
                qs.append(int(rng.integers(-20, 300)))
        if poison:
            ts[int(rng.integers(0, len(ts)))] = int(rng.choice([-1, 27, 31, 200]))
        if trial % 11 == 10 and len(ts) > 1:
            ts, qs = ts[:-1], qs[:-1]  # list runs out
        raw_t, raw_q = np.array(ts, np.int32), np.array(qs, np.int32)
        want = _place_reference(w, h, len(ts), raw_t, raw_q)
        tm, rq = np.zeros((h, w), np.uint8), np.zeros((h, w), np.int32)
        r = lib.jxo_t_place_varblocks(w, h, len(ts), raw_t.ctypes.data, raw_q.ctypes.data, tm.ctypes.data, rq.ctypes.data)
        if want is None:
            assert r != 0, trial
            bad += 1
        else:
            assert r == 0, trial
            assert np.array_equal(tm, want[0]) and np.array_equal(rq, want[1]), trial
            ok += 1
    assert ok > 150 and bad > 40, (ok, bad)
