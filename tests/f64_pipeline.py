"""Float64 restatement of the VarDCT float path, written from the reference text (not a test module).

Input: a JxgFrameDesc (ParsedFrame.desc) and the dense coefficient tap [groups][3][65536] i32 - the same array from the
oracle (decode_file(..., taps=True)["coeffs"]) and from the GPU (Batch.read_coeffs). Three stages, each usable on its own
so that an implementation can be checked one stage at a time with its own input:

  A  coefficients -> XYB planes [3][yb*8][xb*8]   frame/group.rs:85-236,454-613, jxl_transforms/src/transform.rs:14-665
  B  Gaborish, EPF                                render/stages/gaborish.rs, features/epf.rs:54-79, render/stages/epf/
  C  XYB -> linear, output curve, stores         render/stages/xyb.rs:197-241, color/tf.rs:13-44,114-150,268-304,
                                                 381-497, from_linear.rs:97-109 (every curve), stages/convert.rs:574-605,
                                                 739-762,831-857 (u8, u16, f16), render/save.rs (orientation)

Every stage also returns a magnitude M per output sample: the same computation on absolute values (|basis| on |input|,
|weights| on |input|, first-order propagation through the non-linear steps). An f32 implementation of the stage is then
bounded by |got - ref| <= K * 2^-24 * M + 1e-9 with one K per stage (BOUND_K; DESIGN.md section 4).

The only constants read as data are oracle/afv_basis.inc, oracle/dither_table.inc and the parameter literals of the
library's dequantisation matrices. The matrices themselves come from tests/f64_quant.py, the float64 restatement of
quant_weights.rs: the library defaults, or the custom encodings a frame was written with (Frame(d, encodings=...)).
Stage A's M carries the f32 rounding of the implementation's table (f64_quant.K_Q).
"""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 2.0 ** -24
BOUND_K = {"A": 256, "B": 16, "C": 16}  # measured on the oracle and the GPU; DESIGN.md section 4

COV_X = [1, 1, 1, 1, 2, 4, 1, 2, 1, 4, 2, 4, 1, 1, 1, 1, 1, 1, 8, 4, 8, 16, 8, 16, 32, 16, 32]  # transform_map.rs:98-103
COV_Y = [1, 1, 1, 1, 2, 4, 2, 1, 4, 1, 4, 2, 1, 1, 1, 1, 1, 1, 8, 8, 4, 16, 16, 8, 32, 32, 16]  # transform_map.rs:105-110
SPECIAL_8X8 = (1, 2, 3, 12, 13, 14, 15, 16, 17)  # IDENTITY, DCT2X2, DCT4X4, DCT4X8, DCT8X4, AFV0-3
GROUP_BLOCKS = 32      # 256-pixel groups (frame_header.rs group_dim)
COLOR_TILE_BLOCKS = 8  # color_correlation_map.rs: COLOR_TILE_DIM_IN_BLOCKS
MIN_SIGMA = -3.90524291751269967465540850526868  # jxl/src/lib.rs:28
INV_SIGMA_NUM = -1.1715728752538099024           # features/epf.rs:26


def read_inc(name):
    """A generated C table under oracle/ as float64 numbers."""
    text = open(os.path.join(ROOT, "oracle", name)).read()
    body = "\n".join(line.split("//")[0] for line in text.splitlines())
    return np.array([float(v.strip().rstrip("f")) for v in body.split(",") if v.strip()], np.float64)


AFV_BASIS = read_inc("afv_basis.inc").reshape(16, 16)  # [coefficient j][pixel i], transform.rs:34-303
DITHER = read_inc("dither_table.inc").reshape(32, 32)   # convert.rs:19 (the 32 columns before the SIMD padding)


# ---------------------------------------------------------------------------------------------------------------------
# DCT definitions (jxl_transforms/src/tests.rs:23-180)
# ---------------------------------------------------------------------------------------------------------------------
def alpha(u):
    return 1 / np.sqrt(2) if u == 0 else 1.0


def dct_matrix(n):  # tests.rs:23-60 / 62-100
    m = np.zeros((n, n))
    for u in range(n):
        for y in range(n):
            m[u, y] = alpha(u) * np.cos((y + 0.5) * u * np.pi / n) * np.sqrt(2)
    return m


_DCT = {}


def _dct(n):
    if n not in _DCT:
        _DCT[n] = dct_matrix(n)
    return _DCT[n]


def slow_idct2d(inp):  # tests.rs:123-136
    rows, cols = inp.shape
    if rows < cols:
        a = inp.T
    else:
        a = inp.reshape(-1).reshape(cols, rows)
    b = dct_matrix(a.shape[0]).T @ a
    c = b.T
    return dct_matrix(c.shape[0]).T @ c


def scales(n):  # tests.rs:138-147
    i = np.arange(n)
    return np.cos(i / (16 * n) * np.pi) * np.cos(i / (8 * n) * np.pi) * np.cos(i / (4 * n) * np.pi) * n


def slow_reinterpreting_dct2d(inp):  # tests.rs:149-180
    rows, cols = inp.shape
    d1 = dct_matrix(rows) @ inp
    d2 = dct_matrix(cols) @ d1.T
    res = d2.T if rows < cols else d2
    rs, cs = scales(rows), scales(cols)
    if rows < cols:
        res = res / (rs[:, None] * cs[None, :])
    else:
        res = res / (cs[:, None] * rs[None, :])
    return res


def idct_batch(flat, rows, cols, absolute=False):
    """slow_idct2d on N blocks at once: flat (N, rows*cols) in the coefficient layout (min x max, tests.rs:123-136)."""
    mr, mc = _dct(rows), _dct(cols)
    if absolute:
        mr, mc = np.abs(mr), np.abs(mc)
    lo, hi = min(rows, cols), max(rows, cols)
    a = flat.reshape(-1, lo, hi)
    x = a if rows < cols else a.transpose(0, 2, 1)  # (N, rows, cols)
    return np.einsum("ur,nuc,cv->nrv", mr, x, mc, optimize=True)


def reinterpreting_dct_batch(lf, absolute=False):
    """slow_reinterpreting_dct2d on N inputs (N, rows, cols); output (N, min, max)."""
    _, rows, cols = lf.shape
    dr, dc = _dct(rows), _dct(cols)
    if absolute:
        dr, dc = np.abs(dr), np.abs(dc)
    d = np.einsum("ur,nrc,vc->nuv", dr, lf, dc, optimize=True)  # Dr . lf . Dc^T
    rs, cs = scales(rows), scales(cols)
    if rows < cols:
        return d / (rs[:, None] * cs[None, :])
    return d.transpose(0, 2, 1) / (cs[:, None] * rs[None, :])


# ---------------------------------------------------------------------------------------------------------------------
# transform_to_pixels (transform.rs:377-665)
# ---------------------------------------------------------------------------------------------------------------------
def _idct_flat(v, rows, cols):
    return slow_idct2d(v.reshape(rows, cols)).reshape(-1)


def _top_block(s, src, dst):  # transform.rs:14-32: 2x2 butterflies of the top s x s corner
    h = s // 2
    for y in range(h):
        for x in range(h):
            c00, c01 = src[y * 8 + x], src[y * 8 + h + x]
            c10, c11 = src[(y + h) * 8 + x], src[(y + h) * 8 + h + x]
            dst[y * 2 * 8 + x * 2] = c00 + c01 + c10 + c11
            dst[y * 2 * 8 + x * 2 + 1] = c00 + c01 - c10 - c11
            dst[(y * 2 + 1) * 8 + x * 2] = c00 - c01 + c10 - c11
            dst[(y * 2 + 1) * 8 + x * 2 + 1] = c00 - c01 - c10 + c11


def special_to_pixels(t, coeffs, lf):
    """One 8x8 varblock of a special type from its definition: 64 coefficients (natural order) and one LF sample."""
    c = np.array(coeffs, np.float64).copy()
    c[0] = lf
    out = c.copy()
    if t == 1:  # IDENTITY, transform.rs:530-571
        b00, b01, b10, b11 = c[0], c[1], c[8], c[9]
        dcs = [b00 + b01 + b10 + b11, b00 + b01 - b10 - b11, b00 - b01 + b10 - b11, b00 - b01 - b10 + b11]
        for y in range(2):
            for x in range(2):
                rs = sum(c[(y + iy * 2) * 8 + x + ix * 2] for iy in range(4) for ix in range(4) if ix or iy)
                centre = dcs[y * 2 + x] - rs * (1.0 / 16.0)
                out[(4 * y + 1) * 8 + 4 * x + 1] = centre
                for iy in range(4):
                    for ix in range(4):
                        if ix == 1 and iy == 1:
                            continue
                        out[(y * 4 + iy) * 8 + x * 4 + ix] = c[(y + iy * 2) * 8 + x + ix * 2] + centre
                out[y * 4 * 8 + x * 4] = c[(y + 2) * 8 + x + 2] + centre
    elif t == 2:  # DCT2X2, transform.rs:572-578
        tmp = c.copy()
        _top_block(2, tmp, out)
        _top_block(4, out, tmp)
        _top_block(8, tmp, out)
    elif t == 3:  # DCT4X4, transform.rs:579-612
        b00, b01, b10, b11 = c[0], c[1], c[8], c[9]
        dcs = [b00 + b01 + b10 + b11, b00 + b01 - b10 - b11, b00 - b01 + b10 - b11, b00 - b01 - b10 + b11]
        for y in range(2):
            for x in range(2):
                blk = np.array([c[(y + iy * 2) * 8 + x + ix * 2] for iy in range(4) for ix in range(4)])
                blk[0] = dcs[y * 2 + x]
                blk = _idct_flat(blk, 4, 4)
                for iy in range(4):
                    out[(y * 4 + iy) * 8 + x * 4:(y * 4 + iy) * 8 + x * 4 + 4] = blk[iy * 4:iy * 4 + 4]
    elif t == 13:  # DCT8X4, transform.rs:613-637
        dcs = [c[0] + c[8], c[0] - c[8]]
        for x in range(2):
            blk = np.array([c[(x + iy * 2) * 8 + ix] for iy in range(4) for ix in range(8)])
            blk[0] = dcs[x]
            blk = _idct_flat(blk, 8, 4)
            for iy in range(8):
                out[iy * 8 + x * 4:iy * 8 + x * 4 + 4] = blk[iy * 4:iy * 4 + 4]
    elif t == 12:  # DCT4X8, transform.rs:638-662
        dcs = [c[0] + c[8], c[0] - c[8]]
        for y in range(2):
            blk = np.array([c[(y + iy * 2) * 8 + ix] for iy in range(4) for ix in range(8)])
            blk[0] = dcs[y]
            blk = _idct_flat(blk, 4, 8)
            out[y * 32:y * 32 + 32] = blk
    elif 14 <= t <= 17:  # AFV0-3, transform.rs:295-374,510-529
        kind = t - 14
        ax, ay = kind & 1, kind // 2
        b00, b01, b10 = c[0], c[1], c[8]
        dcs = [(b00 + b10 + b01) * 4.0, b00 + b10 - b01, b00 - b10]
        co = np.array([c[iy * 2 * 8 + ix * 2] for iy in range(4) for ix in range(4)])
        co[0] = dcs[0]
        blk = co @ AFV_BASIS  # pixel i = sum_j coeff[j] * basis[j][i]
        for iy in range(4):
            sy = 3 - iy if ay else iy
            for ix in range(4):
                sx = 3 - ix if ax else ix
                out[(iy + ay * 4) * 8 + ax * 4 + ix] = blk[sy * 4 + sx]
        co = np.array([c[iy * 2 * 8 + ix * 2 + 1] for iy in range(4) for ix in range(4)])
        co[0] = dcs[1]
        blk = _idct_flat(co, 4, 4)
        for iy in range(4):
            out[(iy + ay * 4) * 8 + (1 - ax) * 4:(iy + ay * 4) * 8 + (1 - ax) * 4 + 4] = blk[iy * 4:iy * 4 + 4]
        co = np.array([c[(1 + iy * 2) * 8 + ix] for iy in range(4) for ix in range(8)])
        co[0] = dcs[2]
        blk = _idct_flat(co, 4, 8)
        out[(1 - ay) * 32:(1 - ay) * 32 + 32] = blk
    else:
        raise ValueError(f"transform {t} is not a special 8x8 type")
    return out


def special_matrix(t):
    """The linear map of special_to_pixels as a (64 pixels, 64 coefficients + 1 LF sample) matrix."""
    m = np.zeros((64, 65))
    for k in range(64):
        e = np.zeros(64)
        e[k] = 1.0
        m[:, k] = special_to_pixels(t, e, 0.0)
    m[:, 64] = special_to_pixels(t, np.zeros(64), 1.0)
    return m


def transform_to_pixels_batch(t, coeffs, lf, mag_coeffs=None, mag_lf=None):
    """N varblocks of type t: coeffs (N, 64*cx*cy) in natural order, lf (N, cy, cx). Returns pixels (N, 8cy, 8cx) and,
    when magnitudes of the inputs are given, the magnitude of each pixel."""
    cx, cy = COV_X[t], COV_Y[t]
    n = coeffs.shape[0]
    if t in SPECIAL_8X8:
        m = special_matrix(t)
        v = np.concatenate([coeffs, lf.reshape(n, 1)], axis=1)
        pix = (v @ m.T).reshape(n, 8, 8)
        if mag_coeffs is None:
            return pix
        mv = np.concatenate([mag_coeffs, mag_lf.reshape(n, 1)], axis=1)
        return pix, (mv @ np.abs(m).T).reshape(n, 8, 8)
    lo, hi = min(cx, cy), max(cx, cy)

    def run(co, l, absolute):
        buf = co.reshape(n, 8 * lo, 8 * hi).copy()
        buf[:, :lo, :hi] = reinterpreting_dct_batch(l, absolute)  # LLF from the LF samples (group.rs:227-236)
        return idct_batch(buf.reshape(n, -1), 8 * cy, 8 * cx, absolute)

    pix = run(coeffs, lf, False)
    if mag_coeffs is None:
        return pix
    return pix, run(mag_coeffs, mag_lf, True)


# ---------------------------------------------------------------------------------------------------------------------
# Frame parameters out of a JxgFrameDesc
# ---------------------------------------------------------------------------------------------------------------------
def _arr(ptr, ctype, shape):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape).copy()


def dequant_table(t, encodings=None):
    """(3, 64*cx*cy) dequantisation matrix of transform type t and its magnitude (f64_quant.table_for_transform)."""
    from tests import f64_quant as fq
    return fq.table_for_transform(t, encodings)


class Frame:
    """The fields of a JxgFrameDesc the float path reads, as numpy arrays (edited by the sensitivity tests).
    encodings: the 17 dequantisation encodings the frame was written with (None: library table), required when the
    descriptor carries custom tables, so that stage A never takes its matrices from the code under test.
    header: the header fields the frame was written with (synth.encode_synthetic's dict; tests/f64_header.py). The
    Gaborish, EPF, colour correlation and opsin parameters and the CfL maps are taken from what it decodes to, and the
    descriptor must hold the same values (this pins the front end's parse). Without it the descriptor must hold the
    defaults: a frame with other values is refused, for the same reason as with encodings."""

    def __init__(self, d, encodings=None, header=None):
        from tests import f64_header as fh
        self.width, self.height = int(d.width), int(d.height)
        self.xb, self.yb = (self.width + 7) // 8, (self.height + 7) // 8
        xb, yb = self.xb, self.yb
        custom = [bool(d.dequant_tables[i]) for i in range(17)]
        if encodings is None and any(custom):
            raise ValueError("the frame has custom dequantisation matrices: pass the encodings it was written with")
        if encodings is not None:
            assert len(encodings) == 17
            want = [e is not None for e in encodings]
            if want != custom:
                raise ValueError(f"custom tables {custom} in the frame, encodings given for {want}")
        self.encodings = encodings
        self.global_scale, self.x_qm_scale, self.b_qm_scale = int(d.global_scale), int(d.x_qm_scale), int(d.b_qm_scale)
        self.lf = np.stack([_arr(d.lf[c], C.c_float, (yb, xb)) for c in range(3)]).astype(np.float64)
        # an LF image computed elsewhere in float64 (tests/f64_prefix.py) may replace lf; lf_mag then carries its own
        # error bound, in units of K_A 2^-24, added to |lf| in stage A's magnitudes
        self.lf_mag = None
        self.transform_map = _arr(d.transform_map, C.c_uint8, (yb, xb))
        self.raw_quant = _arr(d.raw_quant_map, C.c_int32, (yb, xb))
        self.epf_map = _arr(d.epf_map, C.c_uint8, (yb, xb))
        ty, tx = (yb + 7) // 8, (xb + 7) // 8
        self.ytox = _arr(d.ytox_map, C.c_int8, (ty, tx)).astype(np.int32)
        self.ytob = _arr(d.ytob_map, C.c_int8, (ty, tx)).astype(np.int32)
        self.gab = int(d.gab)
        self.epf_iters = int(d.epf_iters)
        self.intensity_target = float(d.intensity_target)
        self.output_tf, self.orientation = int(d.output_tf), int(d.orientation)
        self.output_gamma = float(d.output_gamma)
        self.output_luminances = np.array(list(d.output_luminances), np.float64)
        self.output_format = int(d.output_format)
        self.dequant = {}
        want = fh.decode(header, self.gab, self.epf_iters)
        have = fh.descriptor_values(d)
        bad = fh.differing(want, have)
        if bad and header is None:
            raise ValueError(f"the frame has non-default header fields {bad}: pass the header it was written with")
        assert not bad, f"descriptor fields {bad} differ from the header written: {[(have[k], want[k]) for k in bad]}"
        self.gab_w1, self.gab_w2 = want["gab_w1"], want["gab_w2"]
        self.epf_sharp_lut, self.epf_channel_scale = want["epf_sharp_lut"], want["epf_channel_scale"]
        self.epf_quant_mul, self.epf_border_sad_mul = want["epf_quant_mul"], want["epf_border_sad_mul"]
        self.epf_pass0_sigma_scale, self.epf_pass2_sigma_scale = want["epf_pass0_sigma_scale"], want["epf_pass2_sigma_scale"]
        self.color_factor, self.base_x, self.base_b = want["color_factor"], want["base_x"], want["base_b"]
        self.opsin_inverse_matrix = np.array(list(d.opsin_inverse_matrix), np.float64).reshape(3, 3)  # output colour
        self.written_opsin_matrix = want["opsin_inverse_matrix"].reshape(3, 3)
        self.opsin_biases, self.quant_biases = want["opsin_biases"], want["quant_biases"]
        maps = fh.cfl_maps(header, ty, tx)
        if maps is not None:
            assert np.array_equal(maps[0], self.ytox) and np.array_equal(maps[1], self.ytob), "CfL maps differ from those written"
            self.ytox, self.ytob = maps

    def matrix(self, t):
        """(table, M) of transform type t; sensitivity tests may plant their own in self.dequant."""
        if t not in self.dequant:
            self.dequant[t] = dequant_table(t, self.encodings)
        return self.dequant[t]


# ---------------------------------------------------------------------------------------------------------------------
# Stage A: coefficients -> XYB planes
# ---------------------------------------------------------------------------------------------------------------------
def varblocks(fr):
    """Every varblock in decode order (group.rs:454-613): group index, first block (bx, by) in the frame, transform type
    and offset of its coefficients inside the group's dense array."""
    gxn = (fr.xb + GROUP_BLOCKS - 1) // GROUP_BLOCKS
    gyn = (fr.yb + GROUP_BLOCKS - 1) // GROUP_BLOCKS
    out = []
    for g in range(gxn * gyn):
        x0, y0 = (g % gxn) * GROUP_BLOCKS, (g // gxn) * GROUP_BLOCKS
        sub = fr.transform_map[y0:y0 + GROUP_BLOCKS, x0:x0 + GROUP_BLOCKS]
        ys, xs = np.nonzero(sub >= 128)  # row-major: the raster order of the first blocks
        t = (sub[ys, xs] & 127).astype(np.int64)
        size = 64 * np.array(COV_X)[t] * np.array(COV_Y)[t]
        off = np.concatenate([[0], np.cumsum(size)[:-1]]).astype(np.int64)
        out.append((np.full(len(t), g), xs + x0, ys + y0, t, off))
    return [np.concatenate(a) for a in zip(*out)]


def cfl_tile(b):
    """Colour-correlation tile of a block row or column (group.rs:456,463)."""
    return b // COLOR_TILE_BLOCKS


def stage_a(fr, coeffs):
    """coeffs: [groups][3][65536] i32. Returns (planes, M), each [3][yb*8][xb*8] float64."""
    from tests import f64_quant as fq
    planes = np.zeros((3, fr.yb * 8, fr.xb * 8))
    mag = np.zeros_like(planes)
    g, bx, by, ts, off = varblocks(fr)
    inv_gs = 65536.0 / fr.global_scale  # quantizer.rs inv_global_scale
    x_dm = (1.0 / 1.25) ** (fr.x_qm_scale - 2.0)  # group.rs:395-396
    b_dm = (1.0 / 1.25) ** (fr.b_qm_scale - 2.0)
    bias = fr.quant_biases
    for t in np.unique(ts):
        t = int(t)
        sel = ts == t
        cx, cy = COV_X[t], COV_Y[t]
        n = 64 * cx * cy
        gs, bxs, bys, offs = g[sel], bx[sel], by[sel], off[sel]
        idx = offs[:, None] + np.arange(n)[None, :]
        q = np.stack([coeffs[gs[:, None], c, idx] for c in range(3)]).astype(np.float64)  # (3, N, n)
        # adjust_quant_bias (group.rs:85-96)
        with np.errstate(divide="ignore", invalid="ignore"):
            adj = np.where(np.abs(q) < 2, q * bias[:3, None, None], q - bias[3] / q)
        rq = fr.raw_quant[bys, bxs].astype(np.float64)
        sy = inv_gs / rq  # dequant_block (group.rs:153-156)
        scale = np.stack([sy * x_dm, sy, sy * b_dm])[:, :, None]
        mat, mmat = fr.matrix(t)
        d = adj * mat[:, None, :] * scale
        # |d| for the rounding of d, plus the table's own f32 error, K_q 2^-24 M_table, in units of K_A 2^-24
        md = np.abs(d) * (1.0 + fq.K_Q / BOUND_K["A"] * (mmat / mat)[:, None, :])
        ty, tx = cfl_tile(bys), cfl_tile(bxs)
        x_cc = (fr.base_x + fr.ytox[ty, tx] / fr.color_factor)[:, None]  # color_correlation_map.rs:76-88
        b_cc = (fr.base_b + fr.ytob[ty, tx] / fr.color_factor)[:, None]
        deq = np.stack([x_cc * d[1] + d[0], d[1], b_cc * d[1] + d[2]])  # dequant_lane (group.rs:128-129)
        # f32 x_cc = fl(base + fl(map / factor)) is off by up to 2^-24 (|map| / factor + |x_cc|): relative to the
        # operands, not to |x_cc|, which a base can cancel (base -0.5, map 43, factor 84: |x_cc| = 0.012, operands
        # 0.51). The |x_cc| part is inside K_A |x_cc| M_y; the operand part is added, twice, in units of K_A 2^-24.
        ax_cc = np.abs(x_cc) + 2.0 / BOUND_K["A"] * (abs(fr.base_x) + np.abs(fr.ytox[ty, tx]) / fr.color_factor)[:, None]
        ab_cc = np.abs(b_cc) + 2.0 / BOUND_K["A"] * (abs(fr.base_b) + np.abs(fr.ytob[ty, tx]) / fr.color_factor)[:, None]
        mdeq = np.stack([ax_cc * md[1] + md[0], md[1], ab_cc * md[1] + md[2]])
        rows = bys[:, None, None] * 8 + np.arange(8 * cy)[None, :, None]
        cols = bxs[:, None, None] * 8 + np.arange(8 * cx)[None, None, :]
        lrows = bys[:, None, None] + np.arange(cy)[None, :, None]
        lcols = bxs[:, None, None] + np.arange(cx)[None, None, :]
        for c in range(3):
            lf = fr.lf[c][lrows, lcols]  # (N, cy, cx), group.rs:227-235
            mlf = np.abs(lf) if fr.lf_mag is None else np.abs(lf) + fr.lf_mag[c][lrows, lcols]
            pix, m = transform_to_pixels_batch(t, deq[c], lf, mdeq[c], mlf)
            planes[c][rows, cols] = pix
            mag[c][rows, cols] = m
    return planes, mag


# ---------------------------------------------------------------------------------------------------------------------
# Stage B: Gaborish, EPF
# ---------------------------------------------------------------------------------------------------------------------
def filter_input(planes, width, height):
    """The filters see the coded frame only: mirroring happens at the coded width and height (run_stage.rs:127-134),
    not at the edge of the planes padded to whole blocks."""
    return planes[:, :height, :width]


def gaborish_f64(img, w1, w2, mag=None):
    """render/stages/gaborish.rs:20-28 (weights normalised to sum 1) on (3, h, w), mirrored edges.
    Magnitude: the stencil on magnitudes, times 1 + 2 (S / |T| - 1) / K_B with T = 1 + 4 w1 + 4 w2 and
    S = 1 + 4 |w1| + 4 |w2|. The normalised weights w / T are rounded in f32 (gaborish.rs:20-27): fl(fl(1 + 4 w1) +
    4 w2) is off by up to 2^-24 (|1 + 4 w1| + |T|) <= 2^-24 (S + |T|), so each weight is off by (S / |T| + 2) 2^-24
    relative, and the output by that times the stencil on magnitudes. For weights >= 0, S = T and the 3 2^-24 is
    inside K_B; a negative weight adds (S / |T| - 1) 2^-24 M, counted twice."""
    def run(x, absolute):
        p = np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="symmetric")
        h, w = x.shape[1:]
        out = np.empty_like(x)
        for c in range(3):
            tot = 1.0 + 4.0 * w1[c] + 4.0 * w2[c]
            k0, k1, k2 = 1.0 / tot, w1[c] / tot, w2[c] / tot
            if absolute:
                grow = 1.0 + 2.0 * ((1.0 + 4.0 * abs(w1[c]) + 4.0 * abs(w2[c])) / abs(tot) - 1.0) / BOUND_K["B"]
                k0, k1, k2 = abs(k0) * grow, abs(k1) * grow, abs(k2) * grow
            s = lambda dx, dy: p[c, 1 + dy:1 + dy + h, 1 + dx:1 + dx + w]  # noqa: E731
            out[c] = (k0 * s(0, 0) + k1 * (s(0, -1) + s(0, 1) + s(-1, 0) + s(1, 0))
                      + k2 * (s(-1, -1) + s(1, -1) + s(-1, 1) + s(1, 1)))
        return out
    out = run(img, False)
    return out if mag is None else (out, run(mag, True))


OFF0 = [(0, -2), (-1, -1), (0, -1), (1, -1), (-2, 0), (-1, 0), (1, 0), (2, 0), (-1, 1), (0, 1), (1, 1), (0, 2)]  # epf0.rs:182-195
OFF1 = [(0, -1), (-1, 0), (1, 0), (0, 1)]                                                                            # epf1.rs:118-123
PLUS = [(0, -1), (-1, 0), (0, 0), (1, 0), (0, 1)]


def epf_border(ys, xs):
    """Pixels on the first or last row or column of an 8x8 block take epf_border_sad_mul (common.rs:31-41)."""
    return np.isin(ys % 8, (0, 7)) | np.isin(xs % 8, (0, 7))


def epf_stage_f64(stage, img, inv_sigma, channel_scale, sigma_scale, border_sad_mul, mag=None, keep=None):
    """img: (3, h, w) float64. Whole-image mirroring at the edges (render/simple_pipeline/run_stage.rs:127-134 with
    util/mirror.rs:8 = numpy's 'symmetric' padding). With `mag`, also returns the magnitude of each output sample: the
    weighted magnitudes of the inputs, the rounding of the division, and the effect of a SAD error on each weight
    (|inv_sigma * sad_mul| times the SAD computed on magnitudes, times |x_j - out|). keep: per block, the blocks that
    pass through (default: inv_sigma < MIN_SIGMA in float64)."""
    _, h, w = img.shape
    R = 3
    P = np.pad(img, ((0, 0), (R, R), (R, R)), mode="symmetric")
    PM = np.pad(mag, ((0, 0), (R, R), (R, R)), mode="symmetric") if mag is not None else None

    def sh(dx, dy, src=P):
        return src[:, R + dy:R + dy + h, R + dx:R + dx + w]

    offs = OFF0 if stage == 0 else OFF1
    scale = np.asarray(channel_scale, np.float64)[:, None, None]
    sads, msads = [], []
    for ox, oy in offs:
        if stage == 2:  # epf2.rs:84-101: one absolute difference per channel
            s = (np.abs(sh(ox, oy) - sh(0, 0)) * scale).sum(axis=0)
            ms = ((sh(ox, oy, PM) + sh(0, 0, PM)) * scale).sum(axis=0) if mag is not None else None
        else:           # epf0.rs:157-168 / epf1.rs:98-101: plus-shaped sums
            s = sum((np.abs(sh(px, py) - sh(px + ox, py + oy)) * scale).sum(axis=0) for px, py in PLUS)
            ms = (sum(((sh(px, py, PM) + sh(px + ox, py + oy, PM)) * scale).sum(axis=0) for px, py in PLUS)
                  if mag is not None else None)
        sads.append(s)
        msads.append(ms)
    ys, xs = np.mgrid[0:h, 0:w]
    sig = inv_sigma[ys // 8, xs // 8]
    sm = sigma_scale * 1.65
    inv_s = sig * np.where(epf_border(ys, xs), sm * border_sad_mul, sm)
    wts = [np.maximum(s * inv_s + 1.0, 0.0) for s in sads]
    wsum = 1.0 + sum(wts)
    out = (sh(0, 0) + sum(wt[None] * sh(ox, oy) for wt, (ox, oy) in zip(wts, offs))) / wsum[None]
    keep = (sig < MIN_SIGMA if keep is None else keep[ys // 8, xs // 8])[None]  # MIN_SIGMA > sigma passes through
    out = np.where(keep, img, out)
    if mag is None:
        return out
    m = (sh(0, 0, PM) + sum(wt[None] * sh(ox, oy, PM) for wt, (ox, oy) in zip(wts, offs))) / wsum[None] + np.abs(out)
    m = m + sum((np.abs(inv_s) * ms)[None] * np.abs(sh(ox, oy) - out) for ms, (ox, oy) in zip(msads, offs)) / wsum[None]
    return out, np.where(keep, mag, m)


def sigma_image_f64(global_scale, raw_quant, sharpness, quant_mul, sharp_lut):  # features/epf.rs:54-79
    quant_scale = 1.0 / (65536.0 / global_scale)
    sigma_quant = quant_mul / (quant_scale * raw_quant.astype(np.float64) * INV_SIGMA_NUM)
    return 1.0 / np.minimum(sigma_quant * np.asarray(sharp_lut, np.float64)[sharpness], -1e-4)


def pass_through_f32(global_scale, raw_quant, sharpness, quant_mul, sharp_lut):
    """The blocks EPF passes through: MIN_SIGMA > sigma, decided on the sigma the reference computes in f32, in its
    operation order (features/epf.rs:53-75, lib.rs:28). It is a branch: a block whose f64 sigma lies within f32
    rounding of MIN_SIGMA (custom LUTs and quant_mul can put one there) takes the f32 side, as every f32
    implementation does. A LUT entry <= 0 gives sigma_quant * lut >= 0, clamped to -1e-4: 1 / sigma = -1e4."""
    f = np.float32
    quant_scale = f(1.0) / (f(65536.0) / f(global_scale))
    sigma_quant = f(quant_mul) / (quant_scale * raw_quant.astype(f) * f(INV_SIGMA_NUM))
    sigma = np.minimum(sigma_quant * np.asarray(sharp_lut, f)[sharpness], f(-1e-4))
    return f(1.0) / sigma < f(MIN_SIGMA)


def stage_b(fr, planes, mag=None):
    """planes: stage-A output [3][yb*8][xb*8]. Returns the filtered coded frame (3, h, w) and its magnitude."""
    x = filter_input(planes, fr.width, fr.height)
    m = np.abs(x) if mag is None else filter_input(mag, fr.width, fr.height)
    h, w = fr.height, fr.width
    if fr.gab:
        x, m = gaborish_f64(x, fr.gab_w1, fr.gab_w2, m)
    if fr.epf_iters > 0:
        # the sigma of a varblock's first block covers the whole varblock: raw_quant_map holds it on every block
        sig = sigma_image_f64(fr.global_scale, fr.raw_quant, fr.epf_map, fr.epf_quant_mul, fr.epf_sharp_lut)
        keep = pass_through_f32(fr.global_scale, fr.raw_quant, fr.epf_map, fr.epf_quant_mul, fr.epf_sharp_lut)
        stages = ([(0, fr.epf_pass0_sigma_scale)] if fr.epf_iters >= 3 else []) + [(1, 1.0)]
        stages += [(2, fr.epf_pass2_sigma_scale)] if fr.epf_iters >= 2 else []  # frame/render.rs: epf_iters
        for st, ss in stages:
            x, m = epf_stage_f64(st, x, sig, fr.epf_channel_scale, ss, fr.epf_border_sad_mul, m, keep)
    return x[:, :h, :w], m[:, :h, :w]


# ---------------------------------------------------------------------------------------------------------------------
# Stage C: XYB -> linear -> output curve -> store
# ---------------------------------------------------------------------------------------------------------------------
TF_LINEAR, TF_SRGB, TF_GAMMA, TF_BT709, TF_PQ, TF_HLG = 0, 1, 2, 3, 4, 5  # include/jxg.h JXG_TF_*


def _f32(v):
    return np.float32(v).astype(np.float64)


SRGB_P = _f32([-5.135152395e-4, 5.287254571e-3, 3.903842876e-1, 1.474205315, 7.352629620e-1])  # tf.rs:15-30
SRGB_Q = _f32([1.004519624e-2, 3.036675394e-1, 1.340816930, 9.258482155e-1, 2.424867759e-2])
BT709_P = _f32([-9.625309705734253e-2, -2.2635456919670105e-1, 1.935774803161621e1, 5.897886276245117e1,
                2.3947298049926758e1])                                                               # tf.rs:120-136
BT709_Q = _f32([1.0, 1.877663230895996e1, 5.5292449951171875e1, 2.6565317153930664e1, 3.269049823284149e-1])
PQ_P = _f32([1.351392e-2, -1.095778, 5.522776e1, 1.492516e2, 4.838434e1])                        # tf.rs:251-252
PQ_Q = _f32([1.012416, 2.016708e1, 9.26371e1, 1.120607e2, 2.590418e1])
PQ_P_SMALL = _f32([9.863406e-6, 3.881234e-1, 1.352821e2, 6.889862e4, -2.864824e5])               # tf.rs:253-260
PQ_Q_SMALL = _f32([3.371868e1, 1.477719e3, 1.608477e4, -4.389884e4, -2.072546e5])
PQ_M1, PQ_M2 = 2610 / 16384, 2523 / 4096 * 128
PQ_C1, PQ_C2, PQ_C3 = 3424 / 4096, 2413 / 4096 * 32, 2392 / 4096 * 32


def rational_poly(x, p, q):
    """util/rational_poly.rs:13-17: p[0] + p[1] x + ... over q[0] + q[1] x + ..., Horner from the top."""
    yp = np.zeros_like(x)
    yq = np.zeros_like(x)
    for a, b in zip(p[::-1], q[::-1]):
        yp = yp * x + a
        yq = yq * x + b
    return yp / yq


# The exact curves the reference's approximations stand for (their own tests compare against these, tf.rs:549-705).
def gamma_exact(x, gamma):
    return np.sign(x) * np.abs(x) ** gamma


def bt709_exact(x):
    a = np.abs(x)
    return np.sign(x) * np.where(a < 0.018, 4.5 * a, 1.099 * a ** 0.45 - 0.099)


def pq_exact(x, intensity_target):
    xp = (np.abs(x) * intensity_target / 10000) ** PQ_M1
    return np.sign(x) * ((PQ_C1 + PQ_C2 * xp) / (1 + PQ_C3 * xp)) ** PQ_M2


def hlg_exact(rgb, intensity_target, luminances):
    """Inverse OOTF with the output luminances, then the HLG OETF (tf.rs:381-395,458-470,481-497); rgb (n, 3)."""
    x = np.asarray(rgb, np.float64)
    sg = 1.2 * 1.111 ** np.log2(intensity_target / 1e3)
    e = (1 - sg) / sg
    if abs(e) >= 0.1:
        mixed = x @ np.asarray(luminances, np.float64)
        x = x * (mixed ** e)[:, None]
    a = np.abs(x)
    A = 0.17883277
    B, Cc = 1 - 4 * A, 0.5599107295
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.sign(x) * np.where(a <= 1 / 12, np.sqrt(3 * a), A * np.log(np.maximum(12 * a - B, 1e-30)) + Cc)


def linear_to_srgb_f64(v, mag=None):
    """color/tf.rs:13-44: 12.92 a below 0.0031308, else the rational polynomial of sqrt(a), sign kept. The magnitude
    of the result: |result| (the curve's own roundings) plus the slope of the exact curve times the input's."""
    a = np.abs(v)
    out = np.copysign(np.where(a < 0.0031308, a * 12.92, rational_poly(np.sqrt(a), SRGB_P, SRGB_Q)), v)
    if mag is None:
        return out
    slope = np.where(a < 0.0031308, 12.92, 1.055 / 2.4 * np.maximum(a, 0.0031308) ** (1 / 2.4 - 1))
    return out, np.abs(out) + slope * mag


def linear_to_bt709_f64(v, mag=None):
    """color/tf.rs:114-150: 4.5 a below 0.018, else the rational polynomial of sqrt(a), sign kept; magnitude as for
    sRGB with the slope of 1.099 a^0.45 - 0.099."""
    a = np.abs(v)
    out = np.copysign(np.where(a < 0.018, a * 4.5, rational_poly(np.sqrt(a), BT709_P, BT709_Q)), v)
    if mag is None:
        return out
    slope = np.where(a < 0.018, 4.5, 1.099 * 0.45 * np.maximum(a, 0.018) ** (0.45 - 1))
    return out, np.abs(out) + slope * mag


def linear_to_pq_f64(v, intensity_target, mag=None):
    """color/tf.rs:268-304: the rational polynomial of (a * intensity_target / 10000)^(1/4), a separate one below
    a = 1e-4, sign kept. Magnitude: |result| plus the slope of the exact PQ curve times the input's (the slope grows
    without bound towards 0, so samples near black get a wide bound, as their f32 error does)."""
    a = np.abs(v)
    y_mult = float(np.float32(intensity_target) * np.float32(1 / 10000))
    a14 = np.sqrt(np.sqrt(a * y_mult))
    out = np.copysign(np.where(a < 1e-4, rational_poly(a14, PQ_P_SMALL, PQ_Q_SMALL), rational_poly(a14, PQ_P, PQ_Q)), v)
    if mag is None:
        return out
    ac = np.maximum(a, 1e-12)
    xp = (ac * y_mult) ** PQ_M1
    n, d = PQ_C1 + PQ_C2 * xp, 1 + PQ_C3 * xp
    slope = PQ_M2 * (n / d) ** (PQ_M2 - 1) * (PQ_C2 * d - PQ_C3 * n) / (d * d) * PQ_M1 * xp / ac
    return out, np.abs(out) + np.abs(slope) * mag


LN2 = np.log(2.0)
# CUDA's documented accuracy of the device functions the output curves use (CUDA C Programming Guide, "Mathematical
# Functions"; the library is built without --use_fast_math): log2f 1 ulp, exp2f 2 ulp. One ulp of y is at most 2^-23 |y|,
# i.e. 2 EPS |y|. They enter the magnitudes explicitly: numpy's own functions are more accurate, so a float32 emulation
# alone would set too tight a bar.
ULP_EXP2 = 2 * 2.0   # exp2f: 2 ulp of the result, in EPS |y|
ULP_LOG2 = 2 * 1.0 + 1.0  # log2f: 1 ulp of the log, plus the rounding of the product g * log2 a, in EPS |g log2 a|
# The reference's fast_powf / fast_log2f (util/fast_math.rs:151) are good to about 3e-5 relative: the bar the oracle,
# which restates them, is held to on top of the f32 bound.
FAST_REL = 3e-5
_LOG2_P = _f32([-1.8503833400518310e-6, 1.4287160470083755, 7.4245873327820566e-1])  # fast_math.rs:116-125
_LOG2_Q = _f32([9.9032814277590719e-1, 1.0096718572241148, 1.7409343003366853e-1])
FAST_LOG2_ZERO = _LOG2_P[0] / _LOG2_Q[0] - 127.0  # fast_log2f(+0.0) = -127.0000019
HLG_A = 0.17883277
HLG_B, HLG_C = 1 - 4 * HLG_A, 0.5599107295


def _concave_term(a, m, g, scale=1.0):
    """Propagated error of scale * a^g (0 < g < 1) for an input error K EPS m, in EPS units: the slope at a, but never
    more than (K EPS m)^g (the slope grows without bound at 0, the function's change does not)."""
    kb = BOUND_K["C"] * EPS * m
    with np.errstate(divide="ignore", invalid="ignore"):
        slope = scale * g * np.maximum(a, 1e-300) ** (g - 1) * m
        cap = scale * kb ** g / (BOUND_K["C"] * EPS)
    return np.where(m > 0, np.minimum(slope, cap), 0.0)


def linear_to_gamma_f64(v, g, mag=None):
    """from_linear.rs:97-109 as the kernel computes it: sign(v) |v|^g, exactly (no fast_powf), 0 at 0. Magnitude:
    |y| (1 ulp-terms of exp2f and log2f, the latter scaled by ln2 |g log2 a|) plus the input's through the slope.
    Also returns the oracle's extra allowance: FAST_REL |y|."""
    a = np.abs(v)
    pos = a > 0
    y = np.where(pos, np.where(pos, a, 1.0) ** g, 0.0)
    out = np.copysign(y, v)
    if mag is None:
        return out
    l2 = np.abs(g * np.log2(np.where(pos, a, 1.0)))
    m = y * (ULP_EXP2 + ULP_LOG2 * LN2 * l2) + (_concave_term(a, mag, g) if g < 1 else g * (a + mag) ** (g - 1) * mag)
    return out, m, FAST_REL * y


def hlg_exponent(intensity_target):
    """color/tf.rs:437-445 hlg_display_to_scene in float32, as the front-end computes it; 0 when |e| < 0.1 skips the
    inverse OOTF (tf.rs:380-382). e < 0 above about 600 nits, e > 0 below about 160."""
    f = np.float32
    sg = f(1.2) * np.power(f(1.111), np.log2(f(intensity_target) / f(1e3)))
    e = (f(1.0) - sg) / sg
    return 0.0 if abs(float(e)) < 0.1 else float(e)


def fast_log2_of_mixed(mixed):
    """The log2 the inverse OOTF takes of the mixed luminance (tf.rs:386, fast_log2f: fast_math.rs:128-137), for the
    sign cases where fast_log2f and log2 part:
      mixed > 0             log2(mixed) (fast_log2f's own error is the oracle's FAST_REL allowance)
      mixed < 0, |m| < 2/3  log2|mixed| + 256: the wrapping subtraction of 0x3f2aaaab carries the sign bit into the
                            exponent (2/3 is where that subtraction changes sign: 0x3f2aaaab is the bits of 2/3)
      mixed < 0, |m| >= 2/3 log2|mixed| - 256
      mixed = +0            fast_log2f(0) = P0 / Q0 - 127 (the mantissa comes out as 1.0)
      mixed = -0            the same + 256
    Plain log2 is NaN for all the non-positive cases."""
    a = np.abs(mixed)
    neg = np.signbit(mixed)
    with np.errstate(divide="ignore"):
        lg = np.log2(np.where(a > 0, a, 1.0))
    small = np.float32(a).view(np.uint32) < 0x3f2aaaab
    lg = np.where(neg, lg + np.where(small, 256.0, -256.0), lg)
    return np.where(a == 0, FAST_LOG2_ZERO + np.where(neg, 256.0, 0.0), lg)


def linear_to_hlg_f64(rgb, intensity_target, luminances, mag=None):
    """Inverse OOTF with the output luminances (tf.rs:384-391), then the HLG OETF (tf.rs:481-497), both exact: rgb and
    mag (3, h, w). Magnitude of the OOTF factor mult = 2^(e log2 mixed), relative: exp2f and log2f ulps as for gamma,
    plus the rounding of mixed through |e| / |mixed|. Where |mixed| is within the f32 bound of 0 its sign, and with it
    the +256 branch, is not determined by f32 arithmetic: those samples get an infinite magnitude (any finite output).
    OETF: sqrt(3a) up to 1/12 (slope capped as for gamma), a ln(12a - b) + c above (slope 12a / (12a - b), log2f ulp).
    Returns (out, M, oracle allowance, mask of samples with an undetermined sign of mixed)."""
    e = hlg_exponent(intensity_target)
    x = np.asarray(rgb, np.float64)
    mx = np.abs(x) if mag is None else mag
    amb = np.zeros(x.shape[1:], bool)
    if e != 0.0:
        lum = np.asarray(luminances, np.float64)[:, None, None]
        mixed = (x * lum).sum(axis=0)
        mmix = 2.0 * (np.abs(lum) * mx).sum(axis=0)
        L = e * fast_log2_of_mixed(mixed)
        mult = 2.0 ** L
        amb = np.abs(mixed) <= BOUND_K["C"] * EPS * mmix
        with np.errstate(divide="ignore"):
            rel = ULP_EXP2 + ULP_LOG2 * LN2 * np.abs(L) + np.abs(e) * mmix / np.abs(mixed)
        x = x * mult[None]
        mx = np.abs(x) * (1.0 + rel[None]) + mult[None] * mx
        mx = np.where(amb[None], np.inf, mx)
    a = np.abs(x)
    low = a <= 1.0 / 12.0
    arg = np.maximum(12.0 * a - HLG_B, 1e-300)
    y = np.where(low, np.sqrt(3.0 * a), HLG_A * np.log(arg) + HLG_C)
    out = np.copysign(y, x)
    if mag is None:
        return out
    with np.errstate(invalid="ignore"):
        m_low = 2.0 * y + _concave_term(a, mx, 0.5, np.sqrt(3.0))
        m_high = (3.0 * y + HLG_A * LN2 * ULP_LOG2 * np.abs(np.log2(arg)) + HLG_A * (12.0 * a + arg) / arg
                  + 12.0 * HLG_A / arg * mx)
    m = np.where(low, m_low, m_high)
    # the oracle: FAST_REL on mult times the OETF's slope d out / d ln a, and FAST_REL on its log term
    allow = (np.where(low, 0.5 * y, 12.0 * HLG_A * a / arg) * FAST_REL * (e != 0.0)
             + np.where(low, 0.0, FAST_REL * HLG_A * np.abs(np.log(arg))))
    return out, m, allow, amb


def stage_c(fr, xyb, mag=None, full=False):
    """xyb: filtered coded frame (3, h, w). Returns the RGB_F32 output (h, w, 3) of the coded image (orientation 1:
    `orient` turns it) and its magnitude. With full=True also the oracle's extra allowance for the approximate power and
    log of gamma / HLG (0 elsewhere) and the mask of HLG samples whose mixed luminance has no determined sign."""
    if fr.output_tf not in (TF_LINEAR, TF_SRGB, TF_GAMMA, TF_BT709, TF_PQ, TF_HLG):
        raise ValueError(f"output transfer function {fr.output_tf}")
    m_in = np.abs(xyb) if mag is None else mag
    x, y, b = xyb
    mx, my, mb = m_in
    bias_cbrt = np.cbrt(fr.opsin_biases)
    isc = 255.0 / fr.intensity_target  # xyb.rs intensity_scale
    sb = fr.opsin_biases * isc
    l, m, s = y + x - bias_cbrt[0], y - x - bias_cbrt[1], b - bias_cbrt[2]  # xyb.rs:214-217
    ml, mm, ms = my + mx + abs(bias_cbrt[0]), my + mx + abs(bias_cbrt[1]), mb + abs(bias_cbrt[2])
    lms = np.stack([l * l * l * isc + sb[0], m * m * m * isc + sb[1], s * s * s * isc + sb[2]])  # xyb.rs:219-228
    # d(v^3) = 3 v^2 dv, plus the roundings of the products and of the bias sum
    mlms = np.stack([(3 * ml * ml * ml + abs(sb[0])) * isc, (3 * mm * mm * mm + abs(sb[1])) * isc,
                     (3 * ms * ms * ms + abs(sb[2])) * isc])
    mat = fr.opsin_inverse_matrix
    rgb = np.einsum("ij,jhw->ihw", mat, lms)  # xyb.rs:231-233
    mrgb = np.einsum("ij,jhw->ihw", np.abs(mat), mlms)
    allow = np.zeros_like(rgb)
    amb = np.zeros(rgb.shape[1:], bool)
    if fr.output_tf == TF_SRGB:
        rgb, mrgb = linear_to_srgb_f64(rgb, mrgb)
    elif fr.output_tf == TF_BT709:
        rgb, mrgb = linear_to_bt709_f64(rgb, mrgb)
    elif fr.output_tf == TF_PQ:
        rgb, mrgb = linear_to_pq_f64(rgb, fr.intensity_target, mrgb)
    elif fr.output_tf == TF_GAMMA:
        rgb, mrgb, allow = linear_to_gamma_f64(rgb, fr.output_gamma, mrgb)
    elif fr.output_tf == TF_HLG:
        rgb, mrgb, allow, amb = linear_to_hlg_f64(rgb, fr.intensity_target, fr.output_luminances, mrgb)
    out = (rgb.transpose(1, 2, 0), mrgb.transpose(1, 2, 0))
    return out + (allow.transpose(1, 2, 0), amb) if full else out


SRGB_F32_LIMIT = float(np.finfo(np.float32).max) / 4 / float(SRGB_P[-1])


def srgb_f32_overflow(fr, xyb):
    """(h, w, 3) mask of the samples an f32 sRGB curve cannot compute: the rational polynomial of sqrt(a) (tf.rs:13-44,
    degree 4, Horner) overflows f32 where a^2 p4 > FLT_MAX (here: above FLT_MAX / 4), giving +-inf or NaN while the
    f64 ratio tends to 30.3. Only frames with XYB planes of 1e6 and more (coefficient-entry edges, shifted multi-pass
    frames) reach linear values of 1e19; the mask is empty for every other frame and every other curve."""
    if fr.output_tf != TF_SRGB:
        return np.zeros((fr.height, fr.width, 3), bool)
    lin = np.abs(linear_rgb_f64(fr, np.asarray(xyb, np.float64)))
    return lin * lin > SRGB_F32_LIMIT


def linear_rgb_f64(fr, xyb):
    """Stage C up to the output curve: display-referred linear RGB (h, w, 3), for sorting samples into value regions."""
    lin = Frame.__new__(Frame)
    lin.__dict__.update(fr.__dict__)
    lin.output_tf = TF_LINEAR
    return stage_c(lin, xyb)[0]


# ---------------------------------------------------------------------------------------------------------------------
# Orientation (render/save.rs, headers/image_metadata.rs:85-96 display_pixel)
# ---------------------------------------------------------------------------------------------------------------------
def orient(img, o):
    """The coded image (h, w, ...) as the save stage places it for orientation o (0 counts as 1)."""
    t = img.swapaxes(0, 1)
    return {0: img, 1: img, 2: img[:, ::-1], 3: img[::-1, ::-1], 4: img[::-1], 5: t, 6: np.rot90(img, k=-1),
            7: t[::-1, ::-1], 8: np.rot90(img, k=1)}[o]


# ---------------------------------------------------------------------------------------------------------------------
# Stores
# ---------------------------------------------------------------------------------------------------------------------
def u8_store_f64(rgb):
    """convert.rs:574-605: v * 255 + dither[(y + 13 c) % 32][(x + 23 c) % 32], clamped to [0, 255], before rounding."""
    h, w, _ = rgb.shape
    ys, xs = np.mgrid[0:h, 0:w]
    d = np.stack([DITHER[(ys + 13 * c) % 32, (xs + 23 * c) % 32] for c in range(3)], axis=-1)
    return np.clip(rgb * 255.0 + d, 0.0, 255.0)


def u16_store_f64(v):
    """convert.rs:739-762 at bit depth 16: clamp to [0, 1], scale by 65535, round to nearest (ties to even)."""
    return np.rint(np.clip(v, 0.0, 1.0) * 65535.0)


def f16_from_f32(v):
    """util/float16.rs:82-141 f16::from_f32 on float32 values, at bit level; returns the uint16 codes. Normal halves are
    rounded to nearest even (and may overflow to infinity), f32 zeros and subnormals give a signed zero, |v| below
    2^-24 gives zero, and the f16 subnormal range 2^-24 <= |v| < 2^-14 is TRUNCATED, shifting one bit further than
    IEEE (2^-15 becomes 2^-16). Infinities stay infinite, NaN becomes the quiet NaN 0x7e00 with its sign."""
    bits = np.asarray(v, np.float32).view(np.uint32).astype(np.int64)
    sign = ((bits >> 31) & 1) << 15
    exp = (bits >> 23) & 0xFF
    mant = bits & 0x7FFFFF
    unb = exp - 127
    shift = np.clip(-14 - unb, 0, 31)
    sub = (mant | 0x800000) >> (shift + 14)
    h_exp = unb + 15
    h_mant = mant >> 13
    up = (((mant >> 12) & 1) == 1) & (((mant & 0xFFF) != 0) | ((h_mant & 1) == 1))
    h_mant = h_mant + up
    normal = np.where(h_mant > 0x3FF, np.where(h_exp >= 30, 0x1F << 10, (h_exp + 1) << 10), (h_exp << 10) | h_mant)
    code = np.select([exp == 0, exp == 255, unb < -24, unb < -14, unb > 15],
                     [0, np.where(mant == 0, 0x1F << 10, (0x1F << 10) | 0x200), 0, sub, 0x1F << 10], normal)
    return (sign | code).astype(np.uint16)


def f16_value(codes):
    return np.asarray(codes, np.uint16).view(np.float16).astype(np.float64)


def f16_store_f64(v, tf):
    """convert.rs:831-857 with the clamp of frame/render.rs:746-750 ([0, 1] for PQ, [-0.074, 1.1] for HLG), after the
    f32 rounding of the value; returns the decoded half values."""
    v = np.asarray(v, np.float64)
    if tf == TF_PQ:
        v = np.clip(v, 0.0, 1.0)
    elif tf == TF_HLG:
        v = np.clip(v, -0.074, 1.1)
    return f16_value(f16_from_f32(np.float32(v)))


FMT_U8, FMT_RGBA_U8, FMT_F32, FMT_XYB, FMT_U16, FMT_F16 = 0, 1, 2, 3, 4, 5  # include/jxg.h JXG_FORMAT_*


def store(fmt, v, tf):
    """The output samples of the coded image v (h, w, 3), as float64: u8 / u16 codes, decoded halves, or v for f32."""
    if fmt in (FMT_U8, FMT_RGBA_U8):
        return np.rint(u8_store_f64(v))
    if fmt == FMT_U16:
        return u16_store_f64(v)
    if fmt == FMT_F16:
        return f16_store_f64(v, tf)
    return np.asarray(v, np.float64)


def output_values(fmt, got):
    """An output buffer (display orientation) as float64 samples (h, w, 3); RGBA must be opaque (alpha 255)."""
    got = np.asarray(got)
    if fmt == FMT_RGBA_U8:
        assert (got[..., 3] == 255).all(), "RGBA alpha is not 255"
        got = got[..., :3]
    if fmt == FMT_F16:
        return f16_value(got.view(np.uint16) if got.dtype != np.uint16 else got)
    return got.astype(np.float64)


def bound(stage, mag):
    return BOUND_K[stage] * EPS * mag + 1e-9


def check(stage, got, ref, mag, what="", extra=0.0):
    """Asserts the stage bound (plus `extra`, the oracle's allowance for approximate functions); a NaN or infinite
    sample where the reference is finite always fails. The message reports the largest err / (2^-24 M)."""
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    with np.errstate(invalid="ignore"):
        ratio = float(np.nanmax(np.where(np.isfinite(mag), err / (EPS * mag + 1e-300), 0.0))) if err.size else 0.0
        bad = ~(err <= bound(stage, mag) + extra) | (np.isfinite(ref) & ~np.isfinite(got))
    assert not bad.any(), (f"{what} stage {stage}: {int(bad.sum())} of {bad.size} samples outside K={BOUND_K[stage]}; "
                           f"largest err/(2^-24 M) = {ratio:.3g}, largest err = {float(err.max()):.3g}")
    return ratio


def check_output(fmt, got, ref, mag, tf, orientation=1, what="", extra=0.0):
    """An output buffer (display orientation) against stage C of the coded image (ref, mag: (h, w, 3)). F32: the stage
    bound. Integer and half stores: every code must lie between store(ref - b) and store(ref + b), b the stage-C bound
    (plus `extra`) of the sample. Every store is monotone, so this accepts exactly the codes an implementation exact to
    f32 rounding could produce. Returns the largest err / (2^-24 M) (F32) or the number of codes != store(ref)."""
    if fmt == FMT_F32:
        return check("C", got, orient(ref, orientation), orient(mag, orientation), what, orient(extra, orientation)
                     if np.ndim(extra) else extra)
    g = output_values(fmt, got)
    b = bound("C", mag) + extra
    with np.errstate(invalid="ignore"):
        lo, hi = (orient(store(fmt, ref + s * b, tf), orientation) for s in (-1.0, 1.0))
    bad = ~((g >= lo) & (g <= hi))
    assert g.shape == lo.shape, f"{what} format {fmt}: shape {g.shape}, want {lo.shape}"
    assert not bad.any(), (f"{what} format {fmt}: {int(bad.sum())} of {bad.size} samples outside "
                           f"[store(ref - b), store(ref + b)]; first at {np.argwhere(bad)[0].tolist()}: got "
                           f"{g[bad][0]}, allowed [{lo[bad][0]}, {hi[bad][0]}]")
    return int((g != orient(store(fmt, ref, tf), orientation)).sum())


# ---------------------------------------------------------------------------------------------------------------------
# Edge-value frames: a parsed frame whose LF field is overwritten so that the output stage sees chosen linear values
# ---------------------------------------------------------------------------------------------------------------------
BT2100_LUMINANCES = (0.2627, 0.6780, 0.0593)


def edge_targets():
    """Linear display RGB targets, one per 2x2-block cell: black; each sign pattern with a negative channel; a negative
    luminance with positive channels; values above 1; and greys from 1e-7 to 3, 1.25x apart, which put samples on both
    sides of every curve's breakpoint (sRGB 0.0031308, BT.709 0.018, PQ 1e-4, HLG 1/12) and into the f16 subnormals."""
    t = [(0.0, 0.0, 0.0)]
    for k in range(1, 8):
        s = [-1.0 if k >> i & 1 else 1.0 for i in range(3)]
        t += [(0.2 * s[0], 0.1 * s[1], 0.05 * s[2]), (0.02 * s[0], 0.03 * s[1], 0.01 * s[2])]
    t += [(0.3, -0.2, 0.1), (-0.3, 0.05, 0.2), (0.05, -0.04, 0.3)]
    t += [(1.5, 1.2, 1.1), (2.0, 0.5, 0.2)]
    t += [(g, g, g) for g in 1e-7 * 1.25 ** np.arange(78)]
    return np.array(t, np.float64)


def edge_lf(fr, targets, intensity_target, cell=2):
    """LF planes (3, yb, xb) float32 that decode to `targets` (n, 3) on flat blocks, by inverting XYB -> linear
    (xyb.rs:197-241) through the frame's opsin matrix and biases in float64. Targets repeat in cells of cell x cell blocks."""
    isc = 255.0 / intensity_target
    lms = np.linalg.solve(fr.opsin_inverse_matrix, targets.T)  # (3, n)
    cube = (lms - (fr.opsin_biases * isc)[:, None]) / isc
    l, m, s = np.cbrt(cube) + np.cbrt(fr.opsin_biases)[:, None]
    xyb = np.stack([(l - m) / 2, (l + m) / 2, s])
    cy, cx = (fr.yb + cell - 1) // cell, (fr.xb + cell - 1) // cell
    idx = np.arange(cy * cx).reshape(cy, cx) % len(targets)
    idx = np.repeat(np.repeat(idx, cell, 0), cell, 1)[:fr.yb, :fr.xb]
    return np.ascontiguousarray(xyb[:, idx].astype(np.float32))


def edit_desc(d, lf=None, **fields):
    """Overwrites fields of a JxgFrameDesc in place (output_luminances as a 3-sequence); lf: (3, yb, xb) float32 planes,
    which the caller keeps alive while the descriptor is used. Returns the descriptor."""
    for k, v in fields.items():
        if k == "output_luminances":
            for i in range(3):
                d.output_luminances[i] = v[i]
        else:
            setattr(d, k, v)
    if lf is not None:
        for c in range(3):
            d.lf[c] = lf[c].ctypes.data
    return d


# Curves that lift every small value out of the f16 subnormals: the powers 1/2.2 and 1/2.6 and HLG's sqrt at 100 nits
# (the edge targets' smallest grey, 1e-7, maps to 6.6e-4 or more there).
NO_F16_SUBNORMALS = ("gamma2.2", "dci", "hlg100")


def edge_regions(lin, out, tf, luminances):
    """Number of samples in each edge region, from the f64 linear RGB (h, w, 3) and the f64 output `out` of one frame.
    Every region must be non-empty for a frame to keep its edge coverage."""
    a = np.abs(lin)
    neg = lin < -1e-3
    r = {"black": int((a.max(axis=-1) < 1e-5).sum()), "above_1": int((lin > 1.0).sum()),
         "f16_subnormal": int(((np.abs(out) < 2.0 ** -14) & (np.abs(out) > 2.0 ** -24)).sum())}
    for k in range(1, 8):
        want = np.array([bool(k >> i & 1) for i in range(3)])
        r[f"signs{k}"] = int((neg == want).all(axis=-1).sum())
    mixed = lin @ np.asarray(luminances, np.float64)
    r["mixed_neg_with_pos"] = int(((mixed < -1e-3) & (lin > 1e-3).any(axis=-1)).sum())
    bp = {TF_SRGB: 0.0031308, TF_BT709: 0.018, TF_PQ: 1e-4}.get(tf)
    if tf == TF_HLG:  # the OETF's breakpoint, on the output side: sqrt(3 / 12) = 0.5
        a, bp = np.abs(out), 0.5
    if bp is not None:
        r["below_breakpoint"] = int(((a < bp) & (a > bp / 1.5)).sum())
        r["above_breakpoint"] = int(((a >= bp) & (a < bp * 1.5)).sum())
    return r
