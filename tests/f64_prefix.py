"""Float64 references for the prefix decode (not a test module; used by test_prefix_f64.py and test_gpu_prefix_f64.py):

  - the LF image of a token-level frame (synth.encode_vardct_tokens) from its quantised LF integers: dequant_lf
    (frame/modular/mod.rs:837-929) with the frame's ytox_lf / ytob_lf as written, then the adaptive LF smoothing
    (frame/adaptive_lf_smoothing.rs:44-125), with a magnitude per sample for an f32 bound of the K_LF kind;
  - stage A of a frame cut after some of its sections (frame/decode.rs:744-780): groups with passes are the
    f64_pipeline.stage_a of their coefficients, groups without any the 8x upsampled LF image (prefix_ref);
  - TOC permutations of a frame's sections, in the decoder's convention (logical section i is bitstream entry perm[i]).
"""
import numpy as np

from tests import f64_header as fh
from tests import f64_pipeline as fp
from tests import prefix_ref as pr

# f32 roundings of one LF sample, each relative to the magnitude of its operands (DESIGN.md section 4): dequant_lf 8
# (the factor's product, quotient and scaling, q * fac, ytox_lf / factor, base + that, the product with Y, the sum),
# the smoothing stencil 11 (three sums of four, three weights and their products, W_CENTER's own, two sums), the blend
# (sm - mc) f + mc 3, and the gate 2 (the quotient by the LF factor, 3 - 4 gap).
K_LF = 24
GLOBAL_SCALE_DENOM = 65536.0                   # quantizer.rs
LF_QUANT = np.array([1 / 4096.0, 1 / 512.0, 1 / 256.0])  # quant_weights.rs LF_QUANT: LfQuantFactors' defaults
TOKEN_QUANT_LF = 16                            # synth.encode_vardct_tokens writes quant_lf = 16 (and global_scale 1024)
W_SIDE = float(np.float32(0.20345139757231578))  # adaptive_lf_smoothing.rs:14-18, f32 constants
W_CORNER = float(np.float32(0.0334829185968739))
W_CENTER = 1.0 - 4.0 * (W_SIDE + W_CORNER)


def lf_factors(global_scale, quant_lf, lf_quant=LF_QUANT):
    """dequant_lf's and the smoothing's per-channel factors (mod.rs:849-851, frame/mod.rs:361-368), X, Y, B."""
    return np.asarray(lf_quant, np.float64) * (GLOBAL_SCALE_DENOM / (global_scale * quant_lf))


def dequant_lf_f64(qx, qy, qb, global_scale, quant_lf, base_x, ytox_lf, base_b, ytob_lf, color_factor, mul=1.0,
                   lf_quant=LF_QUANT):
    """dequant_lf (mod.rs:837-877) of a 4:4:4 frame in float64: the quantised channels X, Y, B -> the LF planes (3, h, w)
    X, Y, B and their magnitudes (the operands of every product and sum, with the colour-correlation factor's own
    operands |base| and |ytox_lf| / factor)."""
    fac = lf_factors(global_scale, quant_lf, lf_quant) * mul
    in_x, in_y, in_b = (np.asarray(q, np.float64) * f for q, f in zip((qx, qy, qb), fac))
    cx = base_x + ytox_lf / color_factor  # color_correlation_map.rs:76-93 y_to_x_lf / y_to_b_lf
    cb = base_b + ytob_lf / color_factor
    lf = np.stack([in_y * cx + in_x, in_y, in_y * cb + in_b])
    ax = abs(cx) + abs(base_x) + abs(ytox_lf) / color_factor
    ab = abs(cb) + abs(base_b) + abs(ytob_lf) / color_factor
    mag = np.stack([np.abs(in_y) * ax + np.abs(in_x), np.abs(in_y), np.abs(in_y) * ab + np.abs(in_b)])
    return lf, mag


def smooth_lf_f64(lf, mag, dc_factors):
    """adaptive_lf_smoothing (adaptive_lf_smoothing.rs:44-125) on (3, h, w) X, Y, B planes in float64. mag: the
    magnitudes of the input (f32 errors of K_LF 2^-24 mag). Returns the smoothed planes, their magnitudes (the stencil
    on the input magnitudes, the blend, and the gate: f = max(0, 3 - 4 gap) is continuous with slope 4 in gap, so an
    error in gap moves the output by at most 4 |sm - mc| times it, whichever side of the kink either lies) and the
    gate factor f per interior sample (NaN on the border, which passes through)."""
    _, h, w = lf.shape
    f = np.full((h, w), np.nan)
    if h <= 2 or w <= 2:
        return lf.copy(), mag.copy(), f

    def stencil(p, ws, wc, wm):
        side = p[:, :-2, 1:-1] + p[:, 2:, 1:-1] + p[:, 1:-1, :-2] + p[:, 1:-1, 2:]
        corner = p[:, :-2, :-2] + p[:, :-2, 2:] + p[:, 2:, :-2] + p[:, 2:, 2:]
        return corner * wc + side * ws + p[:, 1:-1, 1:-1] * wm

    mc, mmc = lf[:, 1:-1, 1:-1], mag[:, 1:-1, 1:-1]
    sm = stencil(lf, W_SIDE, W_CORNER, W_CENTER)
    msm = stencil(mag, W_SIDE, W_CORNER, abs(W_CENTER)) + stencil(np.abs(lf), W_SIDE, W_CORNER, abs(W_CENTER))
    dcf = np.asarray(dc_factors, np.float64)[:, None, None]
    gap = np.maximum(0.5, (np.abs(mc - sm) / dcf).max(axis=0))
    fac = np.maximum(0.0, 3.0 - 4.0 * gap)
    mgap = ((mmc + msm + np.abs(mc - sm)) / dcf).max(axis=0)
    out, m = lf.copy(), mag.copy()
    out[:, 1:-1, 1:-1] = (sm - mc) * fac + mc
    m[:, 1:-1, 1:-1] = mmc + np.abs(mc) + fac * (msm + mmc + np.abs(sm - mc)) + 4.0 * np.abs(sm - mc) * mgap
    f[1:-1, 1:-1] = fac
    return out, m, f


def token_lf_image(spec, global_scale):
    """The LF image (3, yb, xb) X, Y, B of a token-level frame from spec["lf"], its magnitude and the smoothing gate.
    ytox_lf / ytob_lf, the bases and the colour factor come from the spec's header as written (f64_header.decode), so
    the front end's parse of them is checked too. global_scale: the descriptor's (the writer's 1024)."""
    header = spec.get("header") or {}
    want = fh.decode(header)
    cc = header.get("color", {})
    q = np.asarray(spec["lf"], np.int64)
    lf, mag = dequant_lf_f64(q[0], q[1], q[2], global_scale, TOKEN_QUANT_LF, want["base_x"], cc.get("ytox_lf", 0),
                             want["base_b"], cc.get("ytob_lf", 0), want["color_factor"])
    return smooth_lf_f64(lf, mag, lf_factors(global_scale, TOKEN_QUANT_LF))


def use_lf_image(fr, lf, mag):
    """Puts an f64 LF image (and its K_LF magnitude) into f64_pipeline.Frame fr in place of the descriptor's planes."""
    assert lf.shape == fr.lf.shape
    fr.lf = lf
    fr.lf_mag = mag * (K_LF / fp.BOUND_K["A"])
    return fr


def groups(fr):
    """(gx, gy) of every 256x256 group of Frame fr, in group order."""
    xg, yg = (fr.xb + 31) // 32, (fr.yb + 31) // 32
    return [(g % xg, g // xg) for g in range(xg * yg)]


def stage_a(fr, coeffs, passes, weights8=None):
    """Stage A of a prefix frame: planes [3][yb*8][xb*8] and M. Groups with passes (passes[g] > 0): f64_pipeline.stage_a
    of their coefficients; groups without: prefix_ref.upsample_lf_group of fr.lf, M = s * the largest |lf| + lf_mag
    of the 5x5 window, s the largest absolute sum of the kernel's 25 weights of an output sample. That covers the 25
    products and sums of the convolution (K_A > 25) and, the clamp to the window's range being 1-Lipschitz, the LF
    image's own error."""
    a, ma = fp.stage_a(fr, coeffs)
    kernel = pr.upsample8_kernel(pr.default_weights8() if weights8 is None else weights8)
    s = np.abs(kernel).sum(axis=(2, 3)).max()
    mlf = np.abs(fr.lf) + (0.0 if fr.lf_mag is None else fr.lf_mag)
    window_max = np.ones((8, 8, 5, 5))  # a sum of 25 non-negative samples, clamped to the window's largest
    for g, (gx, gy) in enumerate(groups(fr)):
        if passes[g]:
            continue
        for c in range(3):
            u = pr.upsample_lf_group(fr.lf[c], gx, gy, kernel)
            sl = (c, slice(gy * 256, gy * 256 + u.shape[0]), slice(gx * 256, gx * 256 + u.shape[1]))
            a[sl] = u
            ma[sl] = s * pr.upsample_lf_group(mlf[c], gx, gy, window_max)
    return a, ma


# ---------------------------------------------------------------------------------------------------------------------
# TOC permutations. Logical order: LfGlobal, the LF groups, HfGlobal, then the HF sections pass by pass in group order.
# ---------------------------------------------------------------------------------------------------------------------
def hf_index(num_lf_groups, num_groups, p, g):
    return 2 + num_lf_groups + p * num_groups + g


def perm_from_stored(stored):
    """The permutation (logical section i -> bitstream entry perm[i]) that stores the logical sections in `stored`."""
    perm = np.empty(len(stored), np.int64)
    perm[np.asarray(stored)] = np.arange(len(stored))
    return perm.tolist()


def toc_permutation(kind, num_lf_groups, num_groups, num_passes):
    """Named permutations of a frame's sections; the LF sections and HfGlobal keep their places.
      reverse:     every pass's groups in reverse group order (later groups arrive first)
      interleaved: pass by group: all the passes of group 0, then of group 1, ...
      pass1_first: as interleaved, with each group's pass 1 stored before its pass 0 (needs 2 passes or more)"""
    head = list(range(2 + num_lf_groups))
    hf = lambda p, g: hf_index(num_lf_groups, num_groups, p, g)  # noqa: E731
    if kind == "reverse":
        body = [hf(p, g) for p in range(num_passes) for g in reversed(range(num_groups))]
    elif kind == "interleaved":
        body = [hf(p, g) for g in range(num_groups) for p in range(num_passes)]
    elif kind == "pass1_first":
        assert num_passes >= 2
        body = [hf(p, g) for g in range(num_groups) for p in [1, 0] + list(range(2, num_passes))]
    else:
        raise KeyError(kind)
    return perm_from_stored(head + body)
