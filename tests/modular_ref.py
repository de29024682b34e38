"""Plain-integer restatement of the reference's Modular decode (jxl/src/frame/modular), for lossless 8-bit frames:
MA trees, properties, the 14 predictors, the weighted predictor, make_pixel, group-local and global RCT, the global
palette without delta entries (get_palette_value, with the delta table of tests/golden/modular_delta_palette.json),
global and group-local Squeeze (default and explicit steps, meta channels; the scalar unsqueeze, and separately the
i32 lane form), the channel -> section rules for any channel list (global section, ModularLF and ModularHF streams)
and the i32 -> u8 store. Written from the reference text (line numbers
below) with Python ints and explicit wrap32 / wrap64; it shares no code with the front-end (csrc/host/modular.cc)
or the synthetic writer.

The model decodes *forward*: `Frame.decode` walks every pixel in decoder order, and a residual chooser picks the symbol
a decoder will read there. It records (leaf id, pack_signed(residual)) and the pixel that results, so one run gives
the token-level description the writer serialises (synth.encode_modular_tokens) and the planes and u8 image any
correct decoder must produce. Contexts come from the model's tree walk: a decoder that takes another leaf reads
another cluster (one per leaf) and another predictor.

Ranges. Residuals, offsets, multipliers and samples reach the full i32 range; where the reference wraps (make_pixel's
`as i32`, the wrapping property subtractions, the WP error buffers, jxl_simd's Wrapping<i32> RCT lanes) the model wraps
the same way. Two places are confined instead, because the reference's i64 arithmetic is only defined below a bound:
  * make_pixel (common.rs:85): guess + mul * dec must fit i64. |guess| < 2^35 (predict_one of i32 neighbours plus an
    i32 offset), so the choosers keep |dec| < 2^30 whenever mul >= 2^31; `make_pixel` asserts the bound.
  * the weighted predictor (predict.rs:456-461): `sum * DIVLOOKUP[weight_sum - 1]` must fit i64. With |sample| <= 2^31
    the subpredictors satisfy |p_i| <= P = max(3 * 2^34, 2^34 + (3 * 31 * 2^31 + 2 * 31 * 2^35) / 32) < 2^37: the
    neighbours carry 3 extra bits (|N| <= 2^34, so p0 = W + NE - N reaches 3 * 2^34) and the error terms are i32.
    Because the weights w_i are non-negative and sum to weight_sum, and DIVLOOKUP[k - 1] * k <= 2^24, |sum * div| <= 2^24 * (P + 1/2) < 2^61. So WP channels need no confinement below
    the i32 range; `WpState.predict` asserts the bound on every pixel.
"""
import numpy as np

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
NUM_PREDICTORS = 14


def wrap32(v):
    return ((v + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def wrap64(v):
    return ((v + (1 << 63)) & 0xFFFFFFFFFFFFFFFF) - (1 << 63)


def u32(v):
    return v & 0xFFFFFFFF


def pack_signed(v):  # the inverse of unpack_signed (entropy_coding/decode.rs), v in i32
    return u32(v << 1) if v >= 0 else u32(((-(v + 1)) << 1) | 1)


# ---------------------------------------------------------------------------------------------------------------------
# Trees (tree.rs)
# ---------------------------------------------------------------------------------------------------------------------
class TreeRefused(Exception):
    pass


def link_tree(tree, check=True):
    """Tree::read (tree.rs:284-351) over a BFS node list ("split", property, value) / ("leaf", predictor, offset,
    mul_log, mul_bits): child indices as the reader assigns them (left = nodes so far + pending + 1), leaf ids in
    reading order, and every refusal of the reader and of validate_tree (check=False: links a tree the reader must
    refuse, so that a frame carrying it can still be written with the symbols a decoder would read)."""
    nodes, to_decode, leaf_id, max_property = [], 1, 0, 0
    for n in tree:
        if to_decode == 0:
            raise ValueError("nodes after the tree is complete")
        to_decode -= 1
        if n[0] == "split":
            prop, val = n[1], n[2]
            if prop > 255:
                _refuse(check, "InvalidProperty")
            max_property = max(max_property, prop)
            left = len(nodes) + to_decode + 1
            nodes.append(("split", prop, val, left, left + 1))
            to_decode += 2
        else:
            pred, off, mul_log, mul_bits = n[1], n[2], n[3], n[4]
            if pred >= NUM_PREDICTORS:
                _refuse(check, "InvalidPredictor")
            if mul_log >= 31:
                _refuse(check, "TreeMultiplierTooLarge")
            mul = (mul_bits + 1) << mul_log
            if mul > 0xFFFFFFFF:
                _refuse(check, "TreeMultiplierBitsTooLarge")
            nodes.append(("leaf", pred, off, mul, leaf_id))
            leaf_id += 1
    if to_decode:
        raise ValueError("incomplete tree")
    if check:
        validate_tree(nodes, max_property + 1)
    return nodes, max_property + 1


def _refuse(check, what):
    """check: True raises, a list (a frame written with check=False) collects the refusal, False ignores it."""
    if check is True:
        raise TreeRefused(what)
    if isinstance(check, list):
        check.append(what)


def validate_tree(nodes, num_properties):
    """tree.rs:39-155: a split must satisfy lo <= val < hi for the range [lo, hi] its ancestors leave (left child
    (val + 1, hi), right child (lo, val)); no node deeper than 2048."""
    ranges = [(I32_MIN, I32_MAX)] * num_properties
    stack = [(0, 0, ranges)]
    while stack:
        i, depth, rng = stack.pop()
        if depth > 2048:
            raise TreeRefused("TreeTooTall")
        n = nodes[i]
        if n[0] == "leaf":
            continue
        p, val = n[1], n[2]
        lo, hi = rng[p]
        if lo > val or hi <= val:
            raise TreeRefused("TreeSplitOnEmptyRange")
        left, right = list(rng), list(rng)
        left[p], right[p] = (val + 1, hi), (lo, val)
        stack.append((n[4], depth + 1, right))
        stack.append((n[3], depth + 1, left))


def walk(nodes, props, trace=None):
    """tree.rs:364-390: property > value goes left."""
    i = 0
    while nodes[i][0] == "split":
        _, p, val, left, right = nodes[i]
        go_left = props[p] > val
        if trace is not None:
            trace.add((p, go_left))
        i = left if go_left else right
    return nodes[i]


# ---------------------------------------------------------------------------------------------------------------------
# Prediction (predict.rs)
# ---------------------------------------------------------------------------------------------------------------------
def get_rows(row, top, toptop, x, y, w, faults=()):
    """PredictionData::get_rows (predict.rs:95-126): left, top, toptop, topleft, topright, leftleft, toprightright."""
    left = row[x - 1] if x > 0 else (top[0] if y > 0 else 0)
    t = top[x] if y > 0 else left
    topleft = top[x - 1] if x > 0 and y > 0 else left
    topright = top[x + 1] if x + 1 < w and y > 0 else t
    leftleft = row[x - 2] if x > 1 else left
    tt = toptop[x] if y > 1 else t
    if x + 2 < w and y > 0:
        trr = top[x + 2]
    else:
        trr = t if "avgall_trr_top" in faults else topright
    return left, t, tt, topleft, topright, leftleft, trr


def clamped_gradient(left, top, topleft):  # predict.rs:139-146
    mn, mx = min(left, top), max(left, top)
    if topleft < mn:
        return mx
    if topleft > mx:
        return mn
    return left + top - topleft


def tdiv(a, b):  # Rust integer division truncates toward zero
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def predict_one(p, d, wp_pred, faults=()):
    """predict.rs:148-199."""
    left, top, toptop, topleft, topright, leftleft, trr = d
    if p == 0:
        return 0
    if p == 1:
        return left
    if p == 2:
        return top
    if p == 3:
        return tdiv(top + left, 2)
    if p == 4:  # Select: a tie goes to top
        q = left + top - topleft
        if "select_tie_west" in faults:
            return left if abs(q - left) <= abs(q - top) else top
        return left if abs(q - left) < abs(q - top) else top
    if p == 5:
        return clamped_gradient(left, top, topleft)
    if p == 6:
        return wp_pred
    if p == 7:
        return topright
    if p == 8:
        return topleft
    if p == 9:
        return leftleft
    if p == 10:
        return tdiv(left + topleft, 2)
    if p == 11:
        return tdiv(top + topleft, 2)
    if p == 12:
        return tdiv(top + topright, 2)
    return tdiv(6 * top - 2 * toptop + 7 * left + leftleft + trr + 3 * topright + 8, 16)


DIVLOOKUP = [(1 << 24) // (i + 1) for i in range(64)]  # predict.rs:204-213


def floor_log2(v):
    return v.bit_length() - 1


class WpState:
    """WeightedPredictorState (predict.rs:221-517); `hdr` = (p1c, p2c, p3ca, p3cb, p3cc, p3cd, p3ce, w0, w1, w2, w3)."""

    DEFAULT = (16, 10, 7, 7, 7, 0, 0, 0xD, 0xC, 0xC, 0xC)  # headers/modular.rs:14-60

    def __init__(self, hdr, xsize, faults=()):
        self.hdr = hdr or self.DEFAULT
        self.xsize = xsize
        n = (xsize + 1) * 2
        self.pred_errors = [[0, 0, 0, 0] for _ in range(n)]
        self.error = [0] * n
        self.prediction = [0, 0, 0, 0]
        self.pred = 0
        self.faults = faults

    def predict(self, x, y, d):
        p1c, p2c, p3ca, p3cb, p3cc, p3cd, p3ce = self.hdr[:7]
        wts = self.hdr[7:]
        cur, prev = (0, self.xsize + 1) if y & 1 else (self.xsize + 1, 0)
        pos_ne = x + 1 if x + 1 < self.xsize else x
        pos_nw = max(x - 1, 0)
        en, ene, enw = self.pred_errors[prev + x], self.pred_errors[prev + pos_ne], self.pred_errors[prev + pos_nw]
        w = []
        for i in range(4):
            s = en[i] + ene[i] + enw[i]
            err = min(s, 0xFFFFFFFF) if "wp_saturate" in self.faults else u32(s)
            shift = max(floor_log2(err + 1) - 5, 0)
            w.append(4 + ((wts[i] * DIVLOOKUP[err >> shift]) >> shift))
        te_w = self.error[cur + x]
        te_n = self.error[prev + 1 + x]
        te_nw = self.error[prev + 1 + pos_nw]
        te_ne = self.error[prev + 1 + pos_ne]
        sum_wn = te_n + te_w
        prop = te_w
        for e in (te_n, te_nw, te_ne):
            if abs(e) > abs(prop):
                prop = e
        left, top, toptop, topleft, topright = d[0], d[1], d[2], d[3], d[4]
        n, wv, ne, nw, nn = top * 8, left * 8, topright * 8, topleft * 8, toptop * 8
        p0 = wv + ne - n
        p1 = n - (((sum_wn + te_ne) * p1c) >> 5)
        p2 = wv - (((sum_wn + te_nw) * p2c) >> 5)
        p3 = n - ((te_nw * p3ca + te_n * p3cb + te_ne * p3cc + (nn - n) * p3cd + (nw - wv) * p3ce) >> 5)
        log_weight = floor_log2(sum(w))
        ws = [wi >> (log_weight - 4) for wi in w]
        weight_sum = sum(ws)
        s = (weight_sum >> 1) - 1 + ws[0] * p0 + ws[1] * p1 + ws[2] * p2 + ws[3] * p3
        prod = s * DIVLOOKUP[weight_sum - 1]
        assert -(1 << 63) <= prod < (1 << 63), "weighted predictor leaves i64"
        pred = prod >> 24
        if ((te_n ^ te_w) | (te_n ^ te_nw)) <= 0:
            pred = max(min(wv, ne, n), min(max(wv, ne, n), pred))
        self.prediction = [p0, p1, p2, p3]
        self.pred = pred
        return (pred + 3) >> 3, wrap32(prop)

    def update(self, val, x, y):
        cur, prev = (0, self.xsize + 1) if y & 1 else (self.xsize + 1, 0)
        v = val * 8
        self.error[cur + x + 1] = wrap32(self.pred - v)
        errs = [u32((abs(p - v) + 3) >> 3) for p in self.prediction]
        self.pred_errors[cur + x] = errs
        pe = self.pred_errors[prev + x + 1]
        for i in range(4):
            s = pe[i] + errs[i]
            pe[i] = min(s, 0xFFFFFFFF) if "wp_saturate" in self.faults else u32(s)


def make_pixel(dec, mul, guess):
    """common.rs:85: (guess + mul * dec) as i32, inside the i64 range the module docstring confines it to."""
    v = guess + mul * dec
    assert wrap64(v) == v
    return wrap32(v)


# ---------------------------------------------------------------------------------------------------------------------
# Channel decode (decode/channel.rs FullTree, common.rs)
# ---------------------------------------------------------------------------------------------------------------------
class Coverage:
    """What a run reached: pixels per predictor, (property, branch) pairs, offset / multiplier leaves, wrapped
    make_pixel results, RCT types; for Squeeze: (tendency branch, clamp, fired) triples, tail columns / rows ("h" /
    "v"), zero-width / zero-height residuals, in_place = false and meta squeezes, the default rules that fired,
    (section kind, shift) pairs of the coded channels, and outputs the `as i32` of unsqueeze wrapped."""

    SQUEEZE_SETS = ("tendency", "tails", "empty_residuals", "default_rules", "sections")

    def __init__(self):
        for k in self.SQUEEZE_SETS:
            setattr(self, k, set())
        self.not_in_place = 0
        self.meta_squeezes = 0
        self.squeeze_wrapped = 0
        self.predictors = set()
        self.branches = set()
        self.offset_leaves = 0
        self.mul_leaves = 0
        self.wrapped = 0
        self.rct = set()
        self.local_rct = set()
        self.ref_slots = set()
        self.palette = set()
        self.wrapped_props = set()

    def merge(self, o):
        self.predictors |= o.predictors
        self.branches |= o.branches
        self.offset_leaves += o.offset_leaves
        self.mul_leaves += o.mul_leaves
        self.wrapped += o.wrapped
        self.rct |= o.rct
        self.local_rct |= o.local_rct
        self.ref_slots |= o.ref_slots
        self.palette |= o.palette
        self.wrapped_props |= o.wrapped_props
        for k in self.SQUEEZE_SETS:
            getattr(self, k).update(getattr(o, k))
        self.not_in_place += o.not_in_place
        self.meta_squeezes += o.meta_squeezes
        self.squeeze_wrapped += o.squeeze_wrapped


def decode_channels(chans, stream_id, tree, wp_hdr, chooser, cov, faults=()):
    """decode_modular_subbitstream's channel loop (bitstream.rs:205-226, channel.rs:125-200) for channels `chans`
    (dicts with w, h, shift and a `data` list of rows to fill). Returns the symbols as (leaf id, u32 value)."""
    nodes, num_props = tree
    if "wp_header_ignored" in faults:
        wp_hdr = None
    num_ref = ((max(num_props - 16, 0) + 3) // 4) * 4
    uses_wp = any(n[0] == "leaf" and n[1] == 6 or n[0] == "split" and n[1] == 15 for n in nodes)
    if "leaf_dfs" in faults:
        nodes = _dfs_leaf_ids(nodes)
    toks = []
    for ci, ch in enumerate(chans):
        w, h = ch["w"], ch["h"]
        ch["data"] = [[0] * w for _ in range(h)]
        if w == 0 or h == 0:
            continue
        wp = WpState(wp_hdr, w, faults) if uses_wp else None
        props = [0] * 512  # room for a split on property 256 (refused by the reader) and its reference slots
        props[0], props[1] = ci, stream_id
        # precompute_references (common.rs:40-82): earlier channels of the same size and shift, nearest first
        order = range(ci - 1, -1, -1) if "refs_farthest_first" not in faults else range(ci)
        key = (lambda o: (o["w"], o["h"])) if "refs_size_only" in faults else (lambda o: (o["w"], o["h"], o["shift"]))
        refs = [chans[j] for j in order if key(chans[j]) == key(ch)]
        refs = refs[:num_ref // 4]
        for y in range(h):
            row, top, toptop = ch["data"][y], ch["data"][y - 1] if y else None, ch["data"][y - 2] if y > 1 else None
            if "prop9_carry" not in faults or y == 0:
                props[9] = 0  # channel.rs:143-146
            props[2] = y
            for x in range(w):
                d = get_rows(row, top, toptop, x, y, w, faults)
                left, t, tt, topleft, topright, leftleft, _ = d
                # compute_properties (tree.rs:189-244)
                props[3] = x
                props[4] = wrap32(abs(t))
                props[5] = wrap32(abs(left))
                props[6] = t
                props[7] = left
                exact = (left - props[9], left + t - topleft, left - topleft, topleft - t, t - topright, t - tt,
                         left - leftleft)  # properties 8..14, wrapping_sub / wrapping_add in the reference
                for k, v in enumerate(exact):
                    props[8 + k] = wrap32(v)
                    if props[8 + k] != v:
                        cov.wrapped_props.add(8 + k)
                wp_pred, props[15] = wp.predict(x, y, d) if wp else (0, 0)
                for k in range(num_ref):
                    props[16 + k] = 0
                for k, rc in enumerate(refs):
                    rr, rp = rc["data"][y], rc["data"][y - 1 if y else 0]
                    v = rr[x]
                    vl = rr[x - 1] if x > 0 else 0
                    vt = rp[x] if y > 0 else vl
                    vtl = rp[x - 1] if x > 0 and y > 0 else vl
                    dv = v - clamped_gradient(vl, vt, vtl)
                    props[16 + 4 * k: 20 + 4 * k] = [wrap32(abs(v)), v, wrap32(abs(dv)), wrap32(dv)]
                    cov.ref_slots.add(k)
                leaf = walk(nodes, props, cov.branches)
                _, pred, off, mul, leaf_id = leaf
                guess = predict_one(pred, d, wp_pred, faults) + off
                dec = chooser(guess, mul, x, y, ci)
                exact = guess + mul * dec
                if "make_pixel_saturate" in faults:
                    val = max(I32_MIN, min(I32_MAX, exact))
                else:
                    val = make_pixel(dec, mul, guess)
                cov.predictors.add(pred)
                cov.offset_leaves += off != 0
                cov.mul_leaves += mul != 1
                cov.wrapped += val != exact
                toks.append((leaf_id, pack_signed(dec)))
                row[x] = val
                if wp:
                    wp.update(val, x, y)
    return toks


def _dfs_leaf_ids(nodes):  # planted fault: leaf ids in depth-first order
    out, ids = list(nodes), {}

    def visit(i):
        if nodes[i][0] == "leaf":
            ids[i] = len(ids)
        else:
            visit(nodes[i][3])
            visit(nodes[i][4])
    visit(0)
    for i, lid in ids.items():
        out[i] = nodes[i][:4] + (lid,)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# RCT (transforms/rct.rs), store (render/stages/convert.rs)
# ---------------------------------------------------------------------------------------------------------------------
def inverse_rct(planes, begin, rct_type, faults=()):
    """do_rct_step (rct.rs:118-157) on three lists of rows, element-wise with Wrapping<i32> lanes (jxl_simd's scalar
    I32Vec is Wrapping<i32>; shr! is an arithmetic shift)."""
    op, perm = rct_type % 7, rct_type // 7
    a, b, c = planes[begin], planes[begin + 1], planes[begin + 2]
    out = ([], [], [])
    for ra, rb, rc in zip(a, b, c):
        o0, o1, o2 = [], [], []
        for v0, v1, v2 in zip(ra, rb, rc):
            if op == 1:
                v2 = wrap32(v2 + v0)
            elif op == 2:
                v1 = wrap32(v1 + v0)
            elif op == 3:
                v1, v2 = wrap32(v1 + v0), wrap32(v2 + v0)
            elif op == 4:
                v1 = wrap32(v1 + (wrap32(v0 + v2) >> 1))
            elif op == 5:
                v2 = wrap32(v0 + v2)
                v1 = wrap32(v1 + (wrap32(v0 + v2) >> 1))
            elif op == 6:
                yy = wrap32(v0 - (v2 >> 1))
                g = wrap32(v2 + yy)
                yy = wrap32(yy - (v1 >> 1))
                r = wrap32(yy + v1)
                v0, v1, v2 = r, g, yy
            o0.append(v0)
            o1.append(v1)
            o2.append(v2)
        out[0].append(o0)
        out[1].append(o1)
        out[2].append(o2)
    r, g, bb = out
    # the buffers are written first and permuted afterwards (rct.rs:127-131): Gbr/Brg are the inverse of libjxl's
    if "rct_gbr_brg_swapped" in faults and perm in (1, 2):
        perm = 3 - perm
    if perm == 1:    # out[1, 2, 0] = in[0, 1, 2]
        g, bb = bb, g
        r, g = g, r
    elif perm == 2:  # out[2, 0, 1] = in[0, 1, 2]
        r, bb = bb, r
        r, g = g, r
    elif perm == 3:
        bb, g = g, bb
    elif perm == 4:
        r, g = g, r
    elif perm == 5:
        r, bb = bb, r
    planes[begin], planes[begin + 1], planes[begin + 2] = r, g, bb


def _delta_palette():
    import json
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "modular_delta_palette.json")
    return json.load(open(path))["delta_palette"]


DELTA_PALETTE = _delta_palette()


def palette_value(pal, index, c, palette_size, bit_depth=8, faults=()):
    """get_palette_value (palette.rs:38-164): negative indices read the delta table (sign from the index parity),
    [size, size + 64) the 4x4x4 cube with its half-step offset, beyond that the 5x5x5 cube (index % 5 per channel,
    so indices past the cube alias back into it), the rest the explicit entries."""
    if index < 0:
        if c >= 3:
            return 0
        i = (-(index + 1)) % (1 + 2 * (len(DELTA_PALETTE) - 1))
        sign = (1 if i & 1 else -1) * (-1 if "palette_negative_sign" in faults else 1)
        r = DELTA_PALETTE[(i + 1) >> 1][c] * sign
        return r * (1 << (bit_depth - 8)) if bit_depth > 8 else r
    scale = lambda v: (v * ((1 << bit_depth) - 1)) >> 2  # noqa: E731  scale::<4> (palette.rs:24-35)
    if palette_size <= index < palette_size + 64:
        if c >= 3:
            return 0
        return scale(((index - palette_size) >> (2 * c)) % 4) + (1 << max(0, bit_depth - 3))
    if index >= palette_size + 64:
        if c >= 3:
            return 0
        i = index - palette_size - 64
        i //= (1, 5, 25)[c] if c < 3 else 1
        return scale(i % 5)
    return pal[c][index]


def inverse_palette(pal, index_plane, num_colors, num_c, cov, faults=()):
    """do_palette_step for num_deltas == 0 and the Zero predictor (palette.rs:165-199): every output sample is the
    palette value of its index."""
    out = []
    for c in range(num_c):
        out.append([[palette_value(pal, v, c, num_colors, 8, faults) for v in row] for row in index_plane])
    for row in index_plane:
        for v in row:
            cov.palette.add("negative" if v < 0 else "explicit" if v < num_colors else "small_cube"
                            if v < num_colors + 64 else "large_cube" if v < num_colors + 64 + 125 else "beyond_cube")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Squeeze (transforms/squeeze.rs, the squeeze arm of meta_apply.rs:90-180)
# ---------------------------------------------------------------------------------------------------------------------
MAX_FIRST_PREVIEW_SIZE = 8


def is_meta(ch):
    return ch["shift"] is None


def default_squeeze(chans, cov, faults=()):
    """squeeze.rs:39-105: the 4:2:0 preview steps when the two channels after the first non-meta one have its size,
    a vertical step first on tall images, then alternating steps until the first channel is at most 8 x 8."""
    nm = 0
    while nm < len(chans) and is_meta(chans[nm]):
        nm += 1
    w, h = chans[nm]["w"], chans[nm]["h"]
    nc = len(chans) - nm
    params = []
    preview = nc >= 2 if "preview_nc2" in faults else nc > 2
    if preview and (chans[nm + 1]["w"], chans[nm + 1]["h"]) == (w, h):
        cov.default_rules.add("preview420")
        if w > 1:
            params.append((True, False, nm + 1, 2))
        if h > 1:
            params.append((False, False, nm + 1, 2))
    if w <= h and h > MAX_FIRST_PREVIEW_SIZE and "no_vertical_first" not in faults:
        cov.default_rules.add("vertical_first")
        params.append((False, True, nm, nc))
        h = -(-h // 2)
    while w > MAX_FIRST_PREVIEW_SIZE or h > MAX_FIRST_PREVIEW_SIZE:
        cov.default_rules.add("alternating")
        if w > MAX_FIRST_PREVIEW_SIZE:
            params.append((True, True, nm, nc))
            w = -(-w // 2)
        if h > MAX_FIRST_PREVIEW_SIZE:
            params.append((False, True, nm, nc))
            h = -(-h // 2)
    return params


def meta_apply_squeeze(chans, steps, cov, check=True, faults=()):
    """The squeeze arm of meta_apply_single_transform on a channel list ({"w", "h", "shift": (hshift, vshift) or None
    for meta channels}), in place: check_squeeze_params (squeeze.rs:17-37), TooManySqueezes (meta_apply.rs:111-113),
    the averages in place of their channels and the residuals after the range (in_place) or at the end. Returns the
    steps applied (default_squeeze's list for an empty one). check=False applies what it can of a refused step, so that
    the frame can still be written."""
    if not steps:
        steps = default_squeeze(chans, cov, faults)
    applied = []
    for hz, in_place, b, n in steps:
        e = b + n
        if n == 0 or e > len(chans):
            _refuse(check, "InvalidChannelRange")
            continue
        if is_meta(chans[b]) != is_meta(chans[e - 1]):
            _refuse(check, "MixingDifferentChannels")
        if is_meta(chans[b]) and not in_place:
            _refuse(check, "MetaSqueezeRequiresInPlace")
        if is_meta(chans[b]):
            cov.meta_squeezes += 1
        if not in_place:
            cov.not_in_place += 1
        off = e if in_place else len(chans)
        for ic in range(n):
            ch = chans[b + ic]
            sh = ch["shift"]
            if sh is not None and (sh[0] > 30 or sh[1] > 30):
                _refuse(check, "TooManySqueezes")
            new = None if sh is None else (sh[0] + 1, sh[1]) if hz else (sh[0], sh[1] + 1)
            w, h = ch["w"], ch["h"]
            if hz:
                avg, res = (-(-w // 2), h), (w - -(-w // 2), h)
            else:
                avg, res = (w, -(-h // 2)), (w, h - -(-h // 2))
            chans[b + ic] = {"w": avg[0], "h": avg[1], "shift": new}
            rshift = sh if "residual_shift_kept" in faults else new
            chans.insert(off + ic, {"w": res[0], "h": res[1], "shift": rshift})
        applied.append((hz, in_place, b, n))
    return applied


def smooth_tendency(b, a, n, cov=None, faults=()):
    """smooth_tendency_scalar (squeeze.rs:143-168) in exact integers: b the output left of / above the pair, a its
    average, n the next average. Records (branch, clamp, fired) in cov.tendency."""
    if b >= a >= n:
        branch = "increasing"
        diff = tdiv(4 * b - 3 * n - a + (5 if "tendency_plus5" in faults else 6), 12)
        clamps = ((lambda d: d - (d & 1) > 2 * (b - a), 2 * (b - a) + 1), (lambda d: d + (d & 1) > 2 * (a - n), 2 * (a - n)))
    elif b <= a <= n:
        branch = "decreasing"
        diff = tdiv(4 * b - 3 * n - a - 6, 12)
        clamps = ((lambda d: d + (d & 1) < 2 * (b - a), 2 * (b - a) - 1), (lambda d: d - (d & 1) < 2 * (a - n), 2 * (a - n)))
    else:
        if cov is not None:
            cov.tendency.add(("none", None, None))
        return 0
    order = (1, 0) if "clamps_swapped" in faults else (0, 1)
    for k in order:
        fired = clamps[k][0](diff)
        if cov is not None:
            cov.tendency.add((branch, k, fired))
        if fired:
            diff = clamps[k][1]
    return diff


def unsqueeze(avg, res, nxt, prev, cov=None, faults=()):
    """unsqueeze_scalar (squeeze.rs:187-194): i64 arithmetic, `diff / 2` truncating toward zero, `as i32` at the end."""
    diff = res + smooth_tendency(prev, avg, nxt, cov, faults)
    a = avg + (diff // 2 if "diff_floor" in faults else tdiv(diff, 2))
    b = a - diff
    wa, wb = wrap32(a), wrap32(b)
    if cov is not None and (wa != a or wb != b):
        cov.squeeze_wrapped += 1
    return wa, wb


def unsqueeze_line(avg, res, cov=None, faults=()):
    """One row of hsqueeze_scalar (squeeze.rs:389-439) or one column of vsqueeze_scalar (576-644) over a whole channel:
    pairs from (avg[x], res[x]) with the next average avg[x + 1] (its own average at the end) and the previous output,
    then the tail avg[-1] when the output length is odd; a channel without residuals is its average
    (do_hsqueeze_step / do_vsqueeze_step shortcuts)."""
    n = len(avg) + len(res)
    if n == 0:
        return []
    if not res:
        return [avg[0]]
    out = [0] * n
    prev = avg[0]
    for x in range(len(res)):
        a, prev = unsqueeze(avg[x], res[x], avg[x + 1] if x + 1 < len(avg) else avg[x], prev, cov, faults)
        out[2 * x], out[2 * x + 1] = a, prev
    if n & 1:
        out[n - 1] = avg[-1]
    return out


def inverse_squeeze(avg, res, horizontal, cov, faults=()):
    """avg, res: lists of rows. Returns the output rows."""
    h, aw = len(avg), len(avg[0]) if avg else 0
    if horizontal:
        rw = len(res[0]) if res else 0
        if rw == 0:
            cov.empty_residuals.add("h")
        out = [unsqueeze_line(avg[y], res[y] if rw else [], cov, faults) for y in range(h)]
        if (aw + rw) & 1 and rw:
            cov.tails.add("h")
            if "tail_wrong_row" in faults:
                for y in range(1, h):
                    out[y][-1] = avg[y - 1][-1]
        return out
    rh = len(res)
    if rh == 0:
        cov.empty_residuals.add("v")
    cols = [unsqueeze_line([r[x] for r in avg], [r[x] for r in res], cov, faults) for x in range(aw)]
    out = [[c[y] for c in cols] for y in range(h + rh)]
    if (h + rh) & 1 and rh:
        cov.tails.add("v")
        if "tail_wrong_row" in faults and h >= 2:
            out[-1] = list(avg[h - 2])
    return out


def undo_squeeze(data, steps, cov, faults=()):
    """The inverse of meta_apply_squeeze on a list of channel planes (lists of rows), last step first."""
    for hz, in_place, b, n in reversed(steps):
        e = b + n
        off = e if in_place else len(data) - n
        for ic in range(n):
            r = off + (n - 1 - ic if "late_offset" in faults and not in_place else ic)
            data[b + ic] = inverse_squeeze(data[b + ic], data[r], hz, cov, faults)
        del data[off:off + n]


def smooth_tendency_lane(a, b, c):
    """smooth_tendency_impl (squeeze.rs:107-141) on one Wrapping<i32> lane (jxl_simd scalar.rs): a the previous
    output, b the average, c the next average; mul_wide_take_high(x, 0x55555556) is (x * 0x55555556) >> 32 in i64,
    abs wraps at i32::MIN, shr! is arithmetic."""
    a_b, b_c, a_c = wrap32(a - b), wrap32(b - c), wrap32(a - c)
    abs_a_b, abs_b_c, abs_a_c = wrap32(abs(a_b)), wrap32(abs(b_c)), wrap32(abs(a_c))
    non_monotonic = (a_b ^ b_c) < 0
    skip = a_b != 0 and non_monotonic
    skip = b_c != 0 and skip
    abs_a_b_3 = wrap32((abs_a_b * 0x55555556) >> 32)
    x = wrap32(2 + abs_a_c + abs_a_b_3) >> 2
    abs_a_b_2_add_x = wrap32(wrap32(abs_a_b << 1) + (x & 1))
    if x > abs_a_b_2_add_x:
        x = wrap32(wrap32(abs_a_b << 1) + 1)
    abs_b_c_2 = wrap32(abs_b_c << 1)
    if wrap32(x + (x & 1)) > abs_b_c_2:
        x = abs_b_c_2
    if skip:
        x = 0
    return wrap32(-x) if a_c < 0 else x


def unsqueeze_lane(avg, res, nxt, prev):
    """unsqueeze_impl (squeeze.rs:170-185) on one lane, every operation wrapping."""
    diff = wrap32(res + smooth_tendency_lane(prev, avg, nxt))
    sign = (diff & 0xFFFFFFFF) >> 31
    a = wrap32(avg + (wrap32(diff + sign) >> 1))
    return a, wrap32(a - diff)


def store_u8(planes):
    """convert.rs ConvertI32ToU8 at bit depth 8: clamp to [0, 255]; grey is replicated into R, G and B."""
    p = np.array(planes, dtype=np.int64)
    if p.shape[0] == 1:
        p = np.repeat(p, 3, axis=0)
    return np.clip(p, 0, 255).astype(np.uint8).transpose(1, 2, 0)


# ---------------------------------------------------------------------------------------------------------------------
# Frames
# ---------------------------------------------------------------------------------------------------------------------
def section_layout(w, h, group_shift, nc):
    """The channel -> section rules (modular/mod.rs:353-400) for nc equal-size channels of shift 0: the leading
    "meta or small" channels go to the global section 0, channels of shift >= 3 to the LF groups (none here), the rest
    to HF group rects. Returns (channels in section 0, HF group rects [(x0, y0, w, h)], number of LF groups)."""
    gd = 128 << group_shift
    n0 = nc if (w <= gd and h <= gd) else 0
    xg, yg = -(-w // gd), -(-h // gd)
    lfd = gd * 8
    n_lf = -(-w // lfd) * -(-h // lfd)
    rects = []
    for g in range(xg * yg):
        x0, y0 = (g % xg) * gd, (g // xg) * gd
        rects.append((x0, y0, min(gd, w - x0), min(gd, h - y0)))
    return n0, rects, n_lf


def grid_rect(ch, dim, gx, gy):
    """get_grid_rect (mod.rs:150-190) of a coded channel in the grid of `dim` image pixels: cells of
    (dim >> hshift) x (dim >> vshift) channel pixels; (x0, y0, w, h), empty past the channel's edge."""
    gw, gh = dim >> ch["shift"][0], dim >> ch["shift"][1]
    bx, by = gx * gw, gy * gh
    if gw == 0 or gh == 0 or bx >= ch["w"] or by >= ch["h"]:
        return (0, 0, 0, 0)
    return (bx, by, min(ch["w"] - bx, gw), min(ch["h"] - by, gh))


def channel_sections(chans, w, h, group_shift, faults=()):
    """The channel -> section rules (mod.rs:341-407, one pass) for any coded channel list: the leading "meta or small"
    channels go to the global section; of the rest, channels with min(hshift, vshift) >= 3 to the ModularLF stream of
    each LF group (stream id 1 + num_lf_groups + g, rects of lf_group_dim >> shift), channels with shift 0..2 to the
    ModularHF stream of each group (rects of group_dim >> shift); meta channels after the first big one go nowhere.
    Returns (n0, [(stream id, [(channel, rect)])] per LF group, the same per HF group)."""
    gd = 128 << group_shift
    lfd = gd * 8
    n0 = 0
    while n0 < len(chans) and (is_meta(chans[n0]) or (chans[n0]["w"] <= gd and chans[n0]["h"] <= gd)):
        n0 += 1
    rest = [i for i in range(n0, len(chans)) if not is_meta(chans[i])]
    xl, yl = -(-w // lfd), -(-h // lfd)
    xg, yg = -(-w // gd), -(-h // gd)
    n_lf = xl * yl
    lf = []
    for g in range(n_lf):
        sid = 1 + n_lf + g + (1 if "lf_stream_id_plus1" in faults else 0)
        lf.append((sid, [(i, grid_rect(chans[i], lfd, g % xl, g // xl)) for i in rest if min(chans[i]["shift"]) >= 3]))
    hf = []
    for g in range(xg * yg):
        hf.append((1 + 3 * n_lf + 17 + g,
                   [(i, grid_rect(chans[i], gd, g % xg, g // xg)) for i in rest if min(chans[i]["shift"]) <= 2]))
    return n0, lf, hf


class Frame:
    """A token-level frame: geometry, global tree and transforms, one description per HF group (WeightedHeader, local
    transforms, local tree). `decode(chooser)` decodes forward and fills .spec (for synth.encode_modular_tokens),
    .planes (the i32 planes before the u8 store, as coded), .u8 (oriented), .cov and .stream_widths (per section, the
    widest channel of its stream: the LZ77 distance multiplier).
    transforms: the global transforms in header order, ("rct", begin, type), ("palette", begin, num_c, num_colors)
    (no delta entries, the Zero predictor: the form the device decodes) or ("squeeze", [(horizontal, in_place, begin,
    num_c), ...]) with [] for the default steps. Without it: `palette` then `global_rct` [(begin, type)].
    palette: None or (num_colors, index_chooser[, begin, num_c]): meta channels take `chooser`, the other channels
    `index_chooser`. groups: group index -> {"wp", "rct": [(begin, type)] or "transforms" (RCT and Squeeze, as above),
    "tree" (local tree or None)}."""

    def __init__(self, w, h, tree, group_shift=1, grey=False, orientation=1, prefix=False, hybrid=(4, 2, 0),
                 global_rct=(), global_wp=None, groups=None, faults=(), check=True, palette=None, transforms=None):
        self.w, self.h, self.tree, self.group_shift, self.grey = w, h, tree, group_shift, grey
        self.orientation, self.prefix, self.hybrid = orientation, prefix, hybrid
        self.global_rct = list(global_rct)
        self.global_wp = global_wp
        self.groups = groups or {}
        self.faults = faults
        self.check = check  # False: write what a decoder must refuse (trees, transform ranges) instead of raising
        self.palette = palette
        self.transforms = transforms

    def _global_transforms(self, nc):
        if self.transforms is not None:
            return list(self.transforms)
        out = []
        if self.palette:
            pb, pn = (self.palette[2], self.palette[3]) if len(self.palette) > 2 else (0, nc)
            out.append(("palette", pb, pn, self.palette[0]))
        return out + [("rct", b, t) for b, t in self.global_rct]

    def _meta_apply(self, chans, transforms, cov):
        """meta_apply_single_transform for each transform; returns (applied transforms, spec dicts)."""
        applied, spec = [], []
        for t in transforms:
            if t[0] == "rct":
                spec.append({"id": 0, "begin": t[1], "rct_type": t[2]})
                if t[2] >= 42:  # headers/modular.rs: rct_type < 42
                    _refuse(self._chk, "InvalidRct")
                _check_equal_channels(chans, t[1], 3, self._chk)
                applied.append(t)
            elif t[0] == "palette":
                _, b, n, ncol = t
                spec.append({"id": 1, "begin": b, "num_c": n, "num_colors": ncol, "num_deltas": 0, "predictor": 0})
                _check_equal_channels(chans, b, n, self._chk)
                info = chans[min(b, len(chans) - 1)]
                del chans[b + 1:b + n]
                chans.insert(0, {"w": ncol, "h": n, "shift": None})
                if b + 1 < len(chans):
                    chans[b + 1] = dict(info)
                applied.append(t)
            else:
                spec.append({"id": 2, "squeezes": list(t[1])})
                applied.append(("squeeze", meta_apply_squeeze(chans, list(t[1]), cov, self._chk, self.faults)))
        return applied, spec

    def decode(self, chooser):
        nc = 1 if self.grey else 3
        gtree = link_tree(self.tree, self.check)
        cov = Coverage()
        self._log = []  # refusals met with check=False
        self._chk = True if self.check else self._log
        chans = [{"w": self.w, "h": self.h, "shift": (0, 0)} for _ in range(nc)]
        applied, gspec = self._meta_apply(chans, self._global_transforms(nc), cov)
        n0, lf, hf = channel_sections(chans, self.w, self.h, self.group_shift, self.faults)
        index_chooser = self.palette[1] if self.palette else chooser
        route = lambda g, m, x, y, c, meta: (chooser if meta else index_chooser)(g, m, x, y, c)  # noqa: E731
        data = [None] * len(chans)
        for i in range(n0):
            cov.sections.add(("global", chans[i]["shift"]))
        s0 = {"use_global_tree": True, "wp": self.global_wp, "transforms": gspec, "tokens": None}
        sc = [dict(chans[i]) for i in range(n0)]
        toks = decode_channels(sc, 0, gtree, self.global_wp,
                               lambda g, m, x, y, c: route(g, m, x, y, c, is_meta(sc[c])), cov, self.faults)
        if any(c["w"] and c["h"] for c in sc):
            s0["tokens"] = toks
        self.stream_widths = [max([c["w"] for c in sc], default=0)]
        for i in range(n0):
            data[i] = sc[i]["data"]
        for i in range(n0, len(chans)):
            data[i] = [[0] * chans[i]["w"] for _ in range(chans[i]["h"])]
        sections = [s0]
        for kind, streams in (("lf", lf), ("hf", hf)):
            for g, (sid, items) in enumerate(streams):
                sections.append(self._group(kind, g, sid, items, chans, data, gtree, route, cov))
                self.stream_widths.append(self._width)
        bad = bool(self._log)
        planes = None
        if not bad:
            for t in reversed(applied):
                if t[0] == "rct":
                    inverse_rct(data, t[1], t[2], self.faults)
                    cov.rct.add(t[2])
                elif t[0] == "palette":
                    _, b, n, ncol = t
                    outs = inverse_palette(data[0], data[b + 1], ncol, n, cov, self.faults)
                    data = data[1:b + 1] + outs + data[b + 2:]
                else:
                    undo_squeeze(data, t[1], cov, self.faults)
            planes = data[:nc]
        self.spec = {"width": self.w, "height": self.h, "group_shift": self.group_shift, "grey": self.grey,
                     "orientation": self.orientation, "prefix": self.prefix, "hybrid": self.hybrid,
                     "tree": self.tree, "sections": sections}
        self.bad = bad
        self.planes = np.array(planes, dtype=np.int64) if planes is not None else None
        from tests.f64_pipeline import orient
        self.u8 = np.ascontiguousarray(orient(store_u8(planes), self.orientation)) if planes is not None else None
        self.cov = cov
        return self

    def _group(self, kind, g, sid, items, chans, data, gtree, route, cov):
        """One ModularLF / ModularHF stream: its rects of the coded channels, the group's local transforms (undone at
        the end of the section, bitstream.rs:230), the symbols; the decoded rects go back into `data`."""
        self._width = 0
        if not any(r[2] and r[3] for _, r in items):
            return None  # bitstream.rs:143-150: no channel with samples, no bytes
        desc = self.groups.get(g, {}) if kind == "hf" else {}
        for i, _ in items:
            cov.sections.add((kind, chans[i]["shift"]))
        local = desc.get("transforms")
        if local is None:
            local = [("rct", b, t) for b, t in desc.get("rct", ())]
        use_global = desc.get("tree") is None
        tree = gtree if use_global else link_tree(desc["tree"], self.check)
        sc = [{"w": r[2], "h": r[3], "shift": chans[i]["shift"]} for i, r in items]
        before = len(self._log)
        applied, lspec = self._meta_apply(sc, local, cov)
        x0s = {k: items[k][1][:2] for k in range(len(items))}
        ch = lambda gg, m, x, y, c: route(gg, m, x + x0s.get(c, (0, 0))[0], y + x0s.get(c, (0, 0))[1], c, False)  # noqa: E731
        toks = decode_channels(sc, sid, tree, desc.get("wp"), ch, cov, self.faults)
        self._width = max(c["w"] for c in sc)
        sec = {"use_global_tree": use_global, "wp": desc.get("wp"), "transforms": lspec, "tree": desc.get("tree"),
               "tokens": toks}
        if len(self._log) > before:
            return sec
        ld = [c["data"] for c in sc]
        for t in reversed(applied):
            if t[0] == "rct":
                inverse_rct(ld, t[1], t[2], self.faults)
                cov.local_rct.add(t[2])
            else:
                undo_squeeze(ld, t[1], cov, self.faults)
        for k, (i, (x0, y0, rw, rh)) in enumerate(items):
            for yy in range(rh):
                data[i][y0 + yy][x0:x0 + rw] = ld[k][yy]
        return sec


def _check_equal_channels(chans, b, n, check):  # meta_apply.rs:26-47
    if b + n > len(chans):
        _refuse(check, "InvalidChannelRange")
        return
    for i in range(1, n):
        if (chans[b + i]["w"], chans[b + i]["h"], chans[b + i]["shift"]) != (chans[b]["w"], chans[b]["h"], chans[b]["shift"]):
            _refuse(check, "MixingDifferentChannels")


# ---------------------------------------------------------------------------------------------------------------------
# Residual choosers and random trees
# ---------------------------------------------------------------------------------------------------------------------
def clamp_dec(dec, mul):
    lim = (1 << 30) if mul >= (1 << 31) else (1 << 31)
    return max(-lim, min(lim - 1, dec))


def picture_chooser(seed, amp=255, p_small=0.1, p_huge=0.0):
    """Residuals toward a smooth target picture of amplitude `amp` (realistic content), with a share of random small
    residuals and of residuals anywhere in the i32 range."""
    rng = np.random.default_rng(seed)

    def choose(guess, mul, x, y, c):
        r = rng.random()
        if r < p_huge:
            return clamp_dec(int(rng.integers(I32_MIN, I32_MAX, endpoint=True)), mul)
        if r < p_huge + p_small:
            return int(rng.integers(-3, 4))
        target = (((x * 7 + y * 3) >> 2) + 40 * c + ((x * y) >> 6)) % 256
        target = target * amp // 255
        return clamp_dec((target - guess) // mul, mul)
    return choose


def index_chooser(seed, num_colors):
    """Palette indices of every kind: explicit entries, the 4x4x4 and 5x5x5 cubes, indices past the 5x5x5 cube up to
    i32::MAX, and negative indices down to i32::MIN (the delta table)."""
    rng = np.random.default_rng(seed)
    n = num_colors

    def choose(guess, mul, x, y, c):
        k = rng.random()
        if k < 0.3:
            t = int(rng.integers(0, n))
        elif k < 0.5:
            t = n + int(rng.integers(0, 64))
        elif k < 0.7:
            t = n + 64 + int(rng.integers(0, 125))
        elif k < 0.8:
            t = int(rng.integers(n + 189, I32_MAX, endpoint=True))
        elif k < 0.95:
            t = -int(rng.integers(1, 300))
        else:
            t = int(rng.integers(I32_MIN, 0))
        return clamp_dec((t - guess) // mul, mul)
    return choose


def random_tree(rng, depth, props, big_values=False, leaf_preds=range(14), wide_leaves=False):
    """A random tree valid under validate_tree, in BFS order: splits on `props`, values drawn inside the range the
    ancestors leave (so both branches can be non-empty), leaves with any predictor, offsets and multipliers."""
    def value_for(p, lo, hi):
        if p == 0:
            cands = [0, 1]
        elif p == 1:
            cands = [0, 20, 40]
        elif p in (2, 3):
            cands = [0, 1, 2, 5, 60, 120]
        elif big_values and rng.random() < 0.3:
            cands = [int(rng.integers(I32_MIN, I32_MAX))]
        else:
            cands = [int(rng.integers(-40, 300))] if p in (4, 5, 6, 7, 16, 17, 20, 21, 24, 25) else [int(rng.integers(-30, 30))]
        cands = [v for v in cands if lo <= v < hi]
        return cands[int(rng.integers(len(cands)))] if cands else None

    def leaf():
        pred = int(rng.choice(list(leaf_preds)))
        if wide_leaves and rng.random() < 0.5:
            r = rng.random()
            if r < 0.3:
                off, ml, mb = int(rng.integers(I32_MIN, I32_MAX, endpoint=True)), 0, 0
            elif r < 0.6:
                ml = int(rng.integers(0, 31))
                mb = int(rng.integers(0, (0xFFFFFFFF >> ml)))  # (mb + 1) << ml <= u32::MAX
                off = int(rng.integers(-1000, 1000))
            else:
                off, ml, mb = int(rng.integers(-5, 6)), int(rng.integers(0, 3)), int(rng.integers(0, 3))
        elif rng.random() < 0.3:
            off, ml, mb = int(rng.integers(-4, 5)), 0, int(rng.integers(0, 2))
        else:
            off, ml, mb = 0, 0, 0
        return ("leaf", pred, off, ml, mb)

    # nested, then BFS
    def build(d, ranges):
        if d == 0 or (d < depth and rng.random() < 0.15):  # the root always splits
            return leaf()
        for _ in range(4):
            p = int(rng.choice(list(props)))
            lo, hi = ranges.get(p, (I32_MIN, I32_MAX))
            v = value_for(p, lo, hi)
            if v is not None:
                break
        else:
            return leaf()
        left, right = dict(ranges), dict(ranges)
        left[p], right[p] = (v + 1, hi), (lo, v)
        return ("split", p, v, build(d - 1, left), build(d - 1, right))

    root = build(depth, {})
    out, queue = [], [root]
    while queue:
        n = queue.pop(0)
        if n[0] == "split":
            out.append(n[:3])
            queue += [n[3], n[4]]
        else:
            out.append(n)
    return out
