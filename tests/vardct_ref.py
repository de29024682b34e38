"""Plain-integer model of the VarDCT HF coefficient decode of jxl-rs, for token-level test frames.

Restated from the reference text, sharing no code with the decoder, the oracle or the synthetic writer:
  - BlockContextMap (block_context_map.rs:61-155): default and custom forms, LF thresholds per channel with the
    bucket of the quantised LF integers (modular/mod.rs dequant_lf: X, then B, then Y, most significant first), qf
    thresholds stored +1 and compared with `qf > t`, block_context with `c < 2 ? c ^ 1 : 2`, nonzero_context,
    zero_density_context with shrc, and the refusals (num_lf_contexts * (nq + 1) > 64, more than 16 block contexts);
  - predict_num_nonzeros (group.rs:70-83) with 32 at (0, 0), one nonzero map per pass and channel holding
    shrc(nonzeros, log_num_blocks);
  - natural coefficient orders (coeff_order.rs:66-120), used_orders selectors 0x5f / 0x13 / 0 / explicit bits, and
    permutations composed as nat[perm[i]] (permutation.rs:92-99) per pass and channel;
  - PassInfo (group.rs:323-378): histogram_index of ceil_log2(num_histograms) bits, refused when >= num_histograms,
    context_offset = histogram_index * num_block_contexts * 495, the shift of each pass;
  - the group loop (group.rs:454-577): first blocks in raster order, channels 1, 0, 2, InvalidNumNonZeros at
    nonzeros + num_blocks > num_coeffs, EndOfBlockResidualNonZeros, `read_signed << shift` with Rust i32 semantics (a
    value that wraps to 0 sets prev = 0 and is not a nonzero), and the dense [groups][3][65536] decode-order output
    summed over passes with i32 wrapping.

The model works forward: a chooser picks every nonzero count and coefficient, the model records the (context, value)
token the decoder will read for it, and synth.encode_vardct_tokens only serialises the result (Frame.spec)."""
import numpy as np

COV_X = [1, 1, 1, 1, 2, 4, 1, 2, 1, 4, 2, 4, 1, 1, 1, 1, 1, 1, 8, 4, 8, 16, 8, 16, 32, 16, 32]
COV_Y = [1, 1, 1, 1, 2, 4, 2, 1, 4, 1, 4, 2, 1, 1, 1, 1, 1, 1, 8, 8, 4, 16, 16, 8, 32, 32, 16]
# coefficient order (0..12) of each transform type: transform_map.rs / coeff_order.rs:23-37
ORDER_OF = [0, 1, 1, 1, 2, 3, 4, 4, 5, 5, 6, 6, 1, 1, 1, 1, 1, 1, 7, 8, 8, 9, 10, 10, 11, 12, 12]
ORDER_LUT = [0, 1, 4, 5, 7, 9, 11, 18, 20, 21, 23, 24, 26]  # TRANSFORM_TYPE_LUT
# block_context_map.rs:20-31
FREQ_CTX = [0xBAD, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 15, 16, 16, 17, 17, 18, 18, 19, 19, 20, 20,
            21, 21, 22, 22, 23, 23, 23, 23, 24, 24, 24, 24, 25, 25, 25, 25, 26, 26, 26, 26, 27, 27, 27, 27, 28, 28, 28,
            28, 29, 29, 29, 29, 30, 30, 30, 30]
NZ_CTX = [0xBAD, 0, 31, 62, 62, 93, 93, 93, 93, 123, 123, 123, 123, 152, 152, 152, 152, 152, 152, 152, 152, 180, 180,
          180, 180, 180, 180, 180, 180, 180, 180, 180, 180, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206,
          206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206]
DEFAULT_BCM = [0, 1, 2, 2, 3, 3, 4, 5, 6, 6, 6, 6, 6, 7, 8, 9, 9, 10, 11, 12, 13, 14, 14, 14, 14, 14, 7, 8, 9, 9, 10,
               11, 12, 13, 14, 14, 14, 14, 14]
NUM_ORDERS = 13
SELECTOR_ORDERS = {0: 0x5F, 1: 0x13, 2: 0}


class DecodeError(Exception):
    """A refusal of the reference; .kind names it like the reference's error."""

    def __init__(self, kind):
        super().__init__(kind)
        self.kind = kind


class Faults:
    """Planted model faults (all off): test_vardct_ref checks that the frame set catches each one."""
    no_c_xor = False            # block_context channel index c instead of c ^ 1 for X / Y
    qf_ge = False               # qf_idx counts raw_quant >= t
    lf_order_xyb = False        # LF bucket of X, Y, B instead of X, B, Y
    pred_no_round = False       # (top + left) / 2 without the + 1
    nz_bucket_63 = False        # the "< 64" boundary of the nonzero bucket at 63
    freq_k_unshifted = False    # FREQ_CTX[k] instead of FREQ_CTX[k >> lnb]
    prev_ge = False             # initial prev with nonzeros >= num_coeffs / 16
    perm_inverted = False       # permutation applied as its inverse
    lehmer_skip0 = False        # permutation composed over the whole order, skip 0 (first blocks permuted too)
    shift_after_prev = False    # prev / nonzero count taken from the value before the shift
    nz_store_floor = False      # nonzero map holds nonzeros >> lnb instead of shrc


F = Faults()


def wrap32(v):
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= 1 << 31 else v


def pack_signed(v):
    return (v << 1) if v >= 0 else ((-(v + 1)) << 1) | 1


def ceil_log2(x):
    n = 0
    while (1 << n) < x:
        n += 1
    return n


def shrc(v, s):  # group.rs: (v + (1 << s) - 1) >> s
    return (v + (1 << s) - 1) >> s


_NAT = {}


def natural_order(o):
    """coeff_order.rs:66-120 for order o."""
    if o in _NAT:
        return _NAT[o]
    t = ORDER_LUT[o]
    cx, cy = COV_X[t], COV_Y[t]
    xsize = cx * 8
    xs = cx // cy
    xsm, xss = xs - 1, ceil_log2(xs)
    out = [0] * (cx * cy * 64)
    cur = cx * cy
    for i in range(xsize):
        for j in range(i + 1):
            x, y = j, i - j
            if i % 2:
                x, y = y, x
            if y & xsm:
                continue
            y >>= xss
            if x < cx and y < cy:
                val = y * cx + x
            else:
                val = cur
                cur += 1
            out[val] = y * xsize + x
    for ir in range(1, xsize):
        i = xsize - ir - 1
        for j in range(i + 1):
            x, y = xsize - 1 - (i - j), xsize - 1 - j
            if i % 2:
                x, y = y, x
            if y & xsm:
                continue
            y >>= xss
            out[cur] = y * xsize + x
            cur += 1
    _NAT[o] = np.asarray(out, np.int64)
    return _NAT[o]


class BlockContextMap:
    """block_context_map.rs:61-155. lf: thresholds of the channels X, Y, B; qf: thresholds as decoded (stored + 1)."""

    def __init__(self, lf=None, qf=None, cmap=None):
        self.default = cmap is None
        self.lf = [list(t) for t in (lf or [[], [], []])]
        self.qf = list(qf or [])
        self.num_lf = 1
        for t in self.lf:
            self.num_lf *= len(t) + 1
        if self.default:
            self.cmap = list(DEFAULT_BCM)
            self.num_ctx = 15
            return
        if self.num_lf * (len(self.qf) + 1) > 64:
            raise DecodeError("BlockContextMapSizeTooBig")
        assert len(cmap) == 39 * self.num_lf * (len(self.qf) + 1)
        self.cmap = list(cmap)
        self.num_ctx = max(self.cmap) + 1
        if self.num_ctx > 16:
            raise DecodeError("TooManyBlockContexts")

    def lf_index(self, qx, qy, qb):
        def bucket(thr, v):
            return sum(1 for t in thr if v > t)
        order = (0, 1, 2) if F.lf_order_xyb else (0, 2, 1)
        vals = (qx, qy, qb)
        b = 0
        for c in order:
            b = b * (len(self.lf[c]) + 1) + bucket(self.lf[c], vals[c])
        return b

    def qf_index(self, raw_quant):
        return sum(1 for t in self.qf if (raw_quant >= t if F.qf_ge else raw_quant > t))

    def block_context(self, c, order, qf_idx, lf_idx):
        ci = (c if F.no_c_xor else c ^ 1) if c < 2 else 2
        idx = ((ci * 13 + order) * (len(self.qf) + 1) + qf_idx) * self.num_lf + lf_idx
        return self.cmap[idx], idx

    def nonzero_context(self, predicted, block_ctx):
        lim = 63 if F.nz_bucket_63 else 64
        nzc = predicted if predicted < 8 else (4 + predicted // 2 if predicted < lim else 36)
        return nzc * self.num_ctx + block_ctx, nzc

    def zero_density_context(self, nonzeros, k, lnb, prev):
        kk = k if F.freq_k_unshifted else k >> lnb
        return (NZ_CTX[shrc(nonzeros, lnb) & 63] + FREQ_CTX[kk & 63]) * 2 + prev

    def spec(self):
        if self.default:
            return None
        return {"lf": self.lf, "qf": self.qf, "map": self.cmap}


def pass_orders(used_orders, perms):
    """The 39 coefficient orders of a pass (order * 3 + channel): natural, composed with perms[(order, c)] when the
    order is used (coeff_order.rs:122-148)."""
    out = {}
    for o in range(NUM_ORDERS):
        nat = natural_order(o)
        for c in range(3):
            perm = perms.get((o, c)) if used_orders & (1 << o) else None
            if perm is None:
                out[3 * o + c] = nat
                continue
            perm = np.asarray(perm, np.int64)
            nb = len(nat) // 64
            if F.lehmer_skip0:  # the coded permutation moved onto the whole order: positions shift by one block
                perm = np.concatenate([perm[nb:], perm[:nb]])
            if F.perm_inverted:
                inv = np.empty_like(perm)
                inv[perm] = np.arange(len(perm))
                perm = inv
            out[3 * o + c] = nat[perm]
    return out


class Frame:
    """One token-level VarDCT frame. varblocks: (bx, by, transform, raw_quant) tiling the frame; lf: (3, yb, xb)
    quantised LF integers X, Y, B; passes: per pass a dict with shift, selector, used_orders, perms, cmap (None: one
    cluster per used block context group), cfgs, log_alpha, prefix, lz77; hist: per (pass, group) histogram index."""

    def __init__(self, width, height, varblocks, lf, bcm, num_histograms, passes, hist):
        self.width, self.height = width, height
        self.xb, self.yb = (width + 7) // 8, (height + 7) // 8
        self.xg, self.yg = (width + 255) // 256, (height + 255) // 256
        self.num_groups = self.xg * self.yg
        self.varblocks = list(varblocks)
        self.lf = np.asarray(lf, np.int64)
        self.bcm = bcm
        self.num_histograms = num_histograms
        self.passes = passes
        self.hist = hist

    def decode(self, chooser):
        """Runs the decode forward. chooser(ev) returns, for ev = dict(pass, group, c, bx, by, t, num_blocks,
        num_coeffs, shift, predicted, ...), (nonzeros, [values from k = num_blocks on]). Sets .tokens, .coeffs,
        .reach, .error (None or the first refusal)."""
        self.error = None
        bcm = self.bcm
        nac = bcm.num_ctx * 495
        first = {}
        for vb in self.varblocks:
            first[(vb[1], vb[0])] = vb
        self.coeffs = np.zeros((self.num_groups, 3, 65536), np.int64)
        self.tokens = [[] for _ in range(len(self.passes) * self.num_groups)]
        reach = {"cells": set(), "nz_buckets": set(), "orders": set(), "shifts": set(), "wrapped": 0, "full": 0,
                 "empty": 0, "last_k": 0, "hist": set(), "lnb": set(), "max_abs": 0}
        self.reach = reach
        orders = [pass_orders(SELECTOR_ORDERS.get(p["selector"], p.get("used_orders", 0)), p.get("perms", {}))
                  for p in self.passes]
        try:
            for g in range(self.num_groups):
                gx, gy = g % self.xg, g // self.xg
                bx0, by0 = gx * 32, gy * 32
                gw, gh = min(32, self.xb - bx0), min(32, self.yb - by0)
                nzmap = [[[0] * 1024 for _ in range(3)] for _ in self.passes]
                hidx = []
                for p in range(len(self.passes)):
                    h = self.hist[p * self.num_groups + g]
                    if h >= self.num_histograms:
                        raise DecodeError("InvalidHistogramIndex")
                    hidx.append(h)
                    reach["hist"].add(h)
                offset = 0
                for by in range(gh):
                    for bx in range(gw):
                        vb = first.get((by0 + by, bx0 + bx))
                        if vb is None:
                            continue
                        t, rq = vb[2], vb[3]
                        cx, cy = COV_X[t], COV_Y[t]
                        nb, nc = cx * cy, cx * cy * 64
                        lnb = ceil_log2(nb)
                        reach["lnb"].add(lnb)
                        o = ORDER_OF[t]
                        qx, qy, qb = (int(self.lf[c, by0 + by, bx0 + bx]) for c in range(3))
                        lf_idx = bcm.lf_index(qx, qy, qb) if bcm.num_lf > 1 else 0
                        qf_idx = bcm.qf_index(rq)
                        for p, ps in enumerate(self.passes):
                            shift = ps["shift"]
                            reach["shifts"].add(shift)
                            toks = self.tokens[p * self.num_groups + g]
                            ctx_off = hidx[p] * nac
                            for c in (1, 0, 2):
                                nz = nzmap[p][c]
                                if bx == 0:
                                    pred = 32 if by == 0 else nz[(by - 1) * 32]
                                elif by == 0:
                                    pred = nz[bx - 1]
                                else:
                                    pred = (nz[(by - 1) * 32 + bx] + nz[by * 32 + bx - 1] + (0 if F.pred_no_round else 1)) // 2
                                bctx, cell = bcm.block_context(c, o, qf_idx, lf_idx)
                                reach["cells"].add(cell)
                                nzctx, bucket = bcm.nonzero_context(pred, bctx)
                                reach["nz_buckets"].add(bucket)
                                ev = dict(p=p, g=g, c=c, bx=bx0 + bx, by=by0 + by, t=t, num_blocks=nb, num_coeffs=nc,
                                          shift=shift, predicted=pred)
                                nonzeros, vals = chooser(ev)
                                toks.append((nzctx + ctx_off, nonzeros))
                                if nonzeros + nb > nc:
                                    raise DecodeError("InvalidNumNonZeros")
                                if nonzeros == nc - nb:
                                    reach["full"] += 1
                                if nonzeros == 0:
                                    reach["empty"] += 1
                                store = (nonzeros >> lnb) if F.nz_store_floor else shrc(nonzeros, lnb)
                                for iy in range(cy):
                                    for ix in range(cx):
                                        nz[(by + iy) * 32 + bx + ix] = store
                                histo = bcm.num_ctx * 37 + 458 * bctx + ctx_off
                                prev = 0 if (nonzeros >= nc // 16 if F.prev_ge else nonzeros > nc // 16) else 1
                                order = orders[p][3 * o + c]
                                reach["orders"].add((p, 3 * o + c, id(order)))
                                k = nb
                                vi = 0
                                while k < nc and nonzeros:
                                    v = vals[vi]
                                    vi += 1
                                    toks.append((histo + bcm.zero_density_context(nonzeros, k, lnb, prev), pack_signed(v)))
                                    coeff = wrap32(v << shift)
                                    if v != 0 and coeff == 0:
                                        reach["wrapped"] += 1
                                    prev = int((v if F.shift_after_prev else coeff) != 0)
                                    nonzeros -= prev
                                    pos = offset + int(order[k])
                                    self.coeffs[g, c, pos] = wrap32(self.coeffs[g, c, pos] + coeff)
                                    reach["max_abs"] = max(reach["max_abs"], abs(int(coeff)))
                                    if nonzeros == 0 and k == nc - 1:
                                        reach["last_k"] += 1
                                    k += 1
                                if nonzeros:
                                    raise DecodeError("EndOfBlockResidualNonZeros")
                        offset += nb * 64
        except DecodeError as e:
            self.error = e.kind
        self.coeffs = self.coeffs.astype(np.int32)
        return self

    @property
    def spec(self):
        sections = []
        for p in range(len(self.passes)):
            for g in range(self.num_groups):
                sections.append((self.hist[p * self.num_groups + g], self.tokens[p * self.num_groups + g]))
        nctx = self.num_histograms * self.bcm.num_ctx * 495
        passes = []
        for ps in self.passes:
            cmap = ps["cmap"](nctx) if callable(ps["cmap"]) else ps["cmap"]
            passes.append({"selector": ps["selector"], "used_orders": ps.get("used_orders", 0),
                           "perms": ps.get("perms", {}), "cmap": list(cmap), "cfgs": ps["cfgs"],
                           "log_alpha": ps.get("log_alpha", 5), "prefix": ps.get("prefix", False),
                           "lz77": ps.get("lz77")})
        return {"width": self.width, "height": self.height, "shifts": [ps["shift"] for ps in self.passes],
                "bcm": self.bcm.spec(), "lf": self.lf, "varblocks": self.varblocks,
                "num_histograms": self.num_histograms, "passes": passes, "sections": sections}
