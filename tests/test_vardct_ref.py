"""The CPU oracle's VarDCT AC coefficient decode against tests/vardct_ref.py, bit for bit, on token-level frames
(synth.encode_vardct_tokens) that reach custom BlockContextMaps with LF and qf thresholds, several histograms,
custom coefficient orders, several passes with shifts, per-cluster hybrid-uint configurations, prefix codes, LZ77 and
every coefficient order. Each frame asserts what it reached; refusals are checked against a valid twin frame, and
planted model faults must each be caught by the frame set."""
import json
import os

import numpy as np
import pytest

from tests import vardct_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ---------------------------------------------------------------------------------------------------------------
# frame construction
# ---------------------------------------------------------------------------------------------------------------
def tile(xb, yb, rng, choices, first=None):
    """Varblocks tiling an xb x yb block frame: at each uncovered block in raster order the first transform of
    `first.get((bx, by))` or of a shuffled `choices` that fits (inside its 32 x 32 group and the frame), else DCT8."""
    cover = np.full((yb, xb), -1, np.int64)
    out = []
    for by in range(yb):
        for bx in range(xb):
            if cover[by, bx] >= 0:
                continue
            cand = list((first or {}).get((bx, by), [])) + [choices[i] for i in rng.permutation(len(choices))] + [0]
            for t in cand:
                cx, cy = R.COV_X[t], R.COV_Y[t]
                if bx + cx > xb or by + cy > yb or bx // 32 != (bx + cx - 1) // 32 or by // 32 != (by + cy - 1) // 32:
                    continue
                if (cover[by:by + cy, bx:bx + cx] >= 0).any():
                    continue
                cover[by:by + cy, bx:bx + cx] = t
                out.append([bx, by, t, int(rng.integers(1, 257))])
                break
    return out


def chooser(seed, vmax=40, p_full=0.05, p_empty=0.1, cap=96, wrap=0.0):
    """Random nonzero counts (empty, full or up to `cap`) and values in [-vmax, vmax] after the pass shift; with
    `wrap`, some zeros are written as values whose shift wraps to 0."""
    rng = np.random.default_rng(seed)

    def choose(ev):
        nb, nc, shift = ev["num_blocks"], ev["num_coeffs"], ev["shift"]
        room = nc - nb
        r = rng.random()
        if r < p_empty:
            nz = 0
        elif r < p_empty + p_full and nc <= 1024:
            nz = room
        else:
            nz = int(rng.integers(1, min(room, cap) + 1))
        if nz == 0:
            return 0, []
        # positions of the nonzeros among the room slots; sometimes the last slot (k = num_coeffs - 1)
        pos = np.sort(rng.choice(room, nz, replace=False)) if nz < room else np.arange(room)
        if nz < room and rng.random() < 0.2:
            pos[-1] = room - 1
            pos = np.unique(pos)
            while len(pos) < nz:
                pos = np.unique(np.concatenate([pos, rng.choice(room, 1)]))
        vals = [0] * (int(pos[-1]) + 1)
        lim = max(1, vmax >> shift)
        for p in pos:
            vals[int(p)] = int(rng.integers(1, lim + 1)) * (1 if rng.random() < 0.5 else -1)
        if wrap and shift:  # zeros written as values whose shift wraps to 0: tokens that are not nonzeros
            for i, v in enumerate(vals):
                if v == 0 and rng.random() < wrap:
                    vals[i] = (1 << (32 - shift)) * int(rng.choice([-1, 1]))
        return nz, vals
    return choose


def cmap_for(num_clusters, salt=0):
    def f(nctx):
        m = [(i * 5 + i // 37 + salt) % num_clusters for i in range(nctx)]
        assert len(set(m)) == num_clusters
        return m
    return f


def lf_field(rng, xb, yb, lo=-30, hi=30):
    return rng.integers(lo, hi + 1, size=(3, yb, xb))


def one_pass(shift=0, clusters=4, cfgs=None, selector=2, used_orders=0, perms=None, log_alpha=6, prefix=False, lz77=None,
             salt=0):
    cfgs = cfgs or [(4, 2, 0)] * clusters
    return {"shift": shift, "selector": selector, "used_orders": used_orders, "perms": perms or {},
            "cmap": cmap_for(len(cfgs), salt), "cfgs": cfgs, "log_alpha": log_alpha, "prefix": prefix, "lz77": lz77}


def order_size(o):
    t = R.ORDER_LUT[o]
    return R.COV_X[t] * R.COV_Y[t] * 64


def perm_kind(o, kind, rng):
    n = order_size(o)
    nb = n // 64
    if kind == "identity":
        return list(range(n))
    if kind == "reversed":
        return list(range(nb)) + list(range(n - 1, nb - 1, -1))
    return list(range(nb)) + (nb + rng.permutation(n - nb)).tolist()


MIXED = [0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17]


def build(name):
    """(Frame, chooser, what the frame must reach)."""
    rng = np.random.default_rng(sum(map(ord, name)) * 7919)
    if name == "default_420":
        xb = yb = 32
        vbs = tile(xb, yb, rng, MIXED)
        f = R.Frame(256, 256, vbs, lf_field(rng, xb, yb), R.BlockContextMap(), 1, [one_pass(clusters=6)], [0])
        return f, chooser(1), {}
    if name == "one_block_context":
        xb, yb = 24, 20
        bcm = R.BlockContextMap([[], [], []], [], [0] * 39)
        f = R.Frame(190, 160, tile(xb, yb, rng, MIXED), lf_field(rng, xb, yb), bcm, 1,
                    [one_pass(cfgs=[(4, 2, 0), (0, 0, 0), (3, 1, 1)], log_alpha=7)], [0])
        return f, chooser(2), {"num_ctx": 1}
    if name in ("lf_x", "lf_y", "lf_b", "lf_all64"):
        thr = {"lf_x": [[-3, 4], [], []], "lf_y": [[], [0, 9, 15], []], "lf_b": [[], [], [-10]],
               "lf_all64": [[-8, 0, 8], [-5, 2, 20], [-1, 0, 1]]}[name]
        xb, yb = 20, 16
        nlf = 1
        for t in thr:
            nlf *= len(t) + 1
        cmap = (np.arange(39 * nlf) * 7 % 16).tolist()
        bcm = R.BlockContextMap(thr, [], cmap)
        cfg = [(4, 2, 0), (2, 1, 0), (5, 2, 1), (0, 0, 0), (4, 0, 0), (6, 3, 3)]
        f = R.Frame(156, 128, tile(xb, yb, rng, MIXED), lf_field(rng, xb, yb, -25, 25), bcm, 1,
                    [one_pass(cfgs=cfg, log_alpha=8)], [0])
        return f, chooser(3), {"num_lf": nlf}
    if name == "qf15":
        qf = [1, 2, 3, 5, 8, 12, 13, 20, 44, 45, 60, 100, 200, 254, 255]
        cmap = (np.arange(39 * 16) * 11 % 16).tolist()
        bcm = R.BlockContextMap([[], [], []], qf, cmap)
        xb, yb = 32, 24
        vbs = tile(xb, yb, rng, MIXED)
        pool = sorted(set(qf + [t + 1 for t in qf if t < 256] + [1, 256]))
        for i, vb in enumerate(vbs):
            vb[3] = pool[i % len(pool)]
        f = R.Frame(256, 192, vbs, lf_field(rng, xb, yb), bcm, 1, [one_pass(clusters=8, log_alpha=7)], [0])
        return f, chooser(4), {"qf_buckets": 16}
    if name in ("hist3", "hist_groups"):
        nh = 3 if name == "hist3" else 4
        xb, yb = 64, 64
        f = R.Frame(512, 512, tile(xb, yb, rng, MIXED), lf_field(rng, xb, yb), R.BlockContextMap(), nh,
                    [one_pass(clusters=8, log_alpha=7)], [0, 2, 1, 2] if nh == 3 else [3, 2, 1, 0])
        return f, chooser(5), {"hist": nh}
    if name == "orders":
        xb, yb = 32, 32
        first = {(0, 0): [5], (8, 0): [4], (16, 0): [9], (24, 0): [8], (0, 8): [11], (16, 8): [10], (0, 16): [7],
                 (8, 16): [6], (16, 16): [1], (17, 16): [12]}
        vbs = tile(xb, yb, rng, MIXED, first)
        perms = {}
        kinds = ["identity", "reversed", "random"]
        for o in range(7):
            for c in range(3):
                perms[(o, c)] = perm_kind(o, kinds[(o + c) % 3], rng)
        p0 = one_pass(shift=1, selector=0, perms=perms, clusters=5)
        perms1 = {(o, c): perm_kind(o, "random", rng) for o in (0, 1, 4) for c in range(3)}
        p1 = one_pass(shift=0, selector=1, perms=perms1, clusters=3, salt=1)
        perms2 = {(o, c): perm_kind(o, kinds[c], rng) for o in (2, 3, 5, 6) for c in range(3)}
        p2 = one_pass(shift=2, selector=3, used_orders=(1 << 2) | (1 << 3) | (1 << 5) | (1 << 6), perms=perms2, salt=2)
        p3 = one_pass(shift=0, selector=2)
        f = R.Frame(256, 256, vbs, lf_field(rng, xb, yb), R.BlockContextMap(), 1, [p0, p1, p2, p3], [0] * 4)
        return f, chooser(6), {"passes": 4}
    if name == "shapes_large":
        xb, yb = 96, 64
        first = {(0, 0): [24], (32, 0): [25], (48, 0): [25], (64, 0): [26], (64, 16): [26], (0, 32): [21],
                 (16, 32): [22], (24, 32): [22], (0, 48): [23], (0, 56): [23], (32, 32): [18], (40, 32): [19],
                 (44, 32): [19], (48, 32): [20], (48, 36): [20]}
        vbs = tile(xb, yb, rng, MIXED, first)
        perms = {(o, c): perm_kind(o, "random", rng) for o in (9, 11, 12) for c in range(3)}
        p = one_pass(selector=3, used_orders=(1 << 9) | (1 << 11) | (1 << 12), perms=perms, clusters=6, log_alpha=7)
        f = R.Frame(768, 512, vbs, lf_field(rng, xb, yb), R.BlockContextMap(), 1, [p], [0] * 6)
        return f, chooser(7, cap=300), {"orders": 13}
    if name == "passes11":
        xb, yb = 16, 12
        shifts = [0, 1, 2, 3, 3, 2, 1, 0, 3, 1, 0]
        ps = [one_pass(shift=s, clusters=2 + i % 3, salt=i) for i, s in enumerate(shifts)]
        f = R.Frame(128, 96, tile(xb, yb, rng, MIXED), lf_field(rng, xb, yb), R.BlockContextMap(), 1, ps, [0] * 11)
        return f, chooser(8, vmax=1 << 20, wrap=0.05), {"passes": 11, "wrapped": True}
    if name == "passes2_wrap":
        xb, yb = 40, 36
        ps = [one_pass(shift=3, clusters=4), one_pass(shift=0, clusters=3, salt=3)]
        f = R.Frame(320, 288, tile(xb, yb, rng, MIXED), lf_field(rng, xb, yb), R.BlockContextMap(), 2, ps,
                    [1, 0, 1, 0, 0, 1, 1, 1])
        return f, chooser(9, vmax=1 << 20, wrap=0.1), {"passes": 2, "wrapped": True}
    if name == "prefix":
        xb, yb = 40, 40
        p = one_pass(cfgs=[(4, 2, 0), (0, 0, 0), (1, 1, 0), (4, 1, 3)], prefix=True)
        f = R.Frame(320, 320, tile(xb, yb, rng, MIXED), lf_field(rng, xb, yb), R.BlockContextMap(), 1, [p], [0] * 4)
        return f, chooser(10), {}
    if name == "lz77":
        xb, yb = 36, 30
        p = one_pass(clusters=3, lz77=(224, 3))
        f = R.Frame(288, 240, tile(xb, yb, rng, MIXED), lf_field(rng, xb, yb), R.BlockContextMap(), 1, [p], [0] * 4)
        return f, chooser(11, p_empty=0.3, vmax=3), {}
    if name == "thin":
        xb, yb = 1, 70
        f = R.Frame(8, 560, tile(xb, yb, rng, MIXED), lf_field(rng, xb, yb), R.BlockContextMap(), 1,
                    [one_pass(clusters=3)], [0] * 3)
        return f, chooser(12, p_full=0.3), {}
    if name == "flat":
        xb, yb = 70, 1
        f = R.Frame(560, 5, tile(xb, yb, rng, MIXED), lf_field(rng, xb, yb), R.BlockContextMap(), 1,
                    [one_pass(clusters=3)], [0] * 3)
        return f, chooser(13, p_full=0.3), {}
    if name == "ragged_tall_wide":
        xb, yb = 33, 35
        first = {(0, 0): [9], (0, 4): [8], (1, 0): [8], (0, 32): [7], (32, 0): [9]}
        f = R.Frame(263, 277, tile(xb, yb, rng, [8, 9, 6, 7, 10, 11, 0], first), lf_field(rng, xb, yb),
                    R.BlockContextMap(), 1, [one_pass(clusters=4)], [0] * 4)
        return f, chooser(14, p_full=0.2, p_empty=0.2), {}
    if name == "entry_edges":
        xb, yb = 32, 32
        vbs = tile(xb, 33, rng, [0], {(0, 0): [24]})
        f = R.Frame(256, 264, vbs, lf_field(rng, xb, 33), R.BlockContextMap(), 1,
                    [one_pass(cfgs=[(4, 2, 0), (0, 0, 0)], log_alpha=8)], [0] * 2)
        return f, edge_chooser(15), {"edges": True}
    raise KeyError(name)


def edge_chooser(seed):
    """Values at both ends of the device's coefficient entry for 8x8 (n = 6: [-2^25, 2^25 - 1]) and 256x256 varblocks
    (n = 16: [-2^15, 2^15 - 1]), plus a full block and a last coefficient at k = num_coeffs - 1."""
    base = chooser(seed, p_full=0.3)

    def choose(ev):
        nc, nb = ev["num_coeffs"], ev["num_blocks"]
        n = (nc).bit_length() - 1
        lo, hi = -(1 << (31 - n)), (1 << (31 - n)) - 1
        if ev["bx"] % 3 == 0 or nc == 65536:
            vals = [lo, hi, 0, 1, -1]
            return 4, vals
        return base(ev)
    return choose


CASES = ["default_420", "one_block_context", "lf_x", "lf_y", "lf_b", "lf_all64", "qf15", "hist3", "hist_groups",
         "orders", "shapes_large", "passes11", "passes2_wrap", "prefix", "lz77", "thin", "flat", "ragged_tall_wide",
         "entry_edges"]

_CACHE = {}


def model(name):
    """(decoded model Frame, file bytes)."""
    if name not in _CACHE:
        import synth
        f, ch, want = build(name)
        f.decode(ch)
        assert f.error is None, (name, f.error)
        _CACHE[name] = (f, synth.encode_vardct_tokens(f.spec), want)
    return _CACHE[name][:2]


def oracle_coeffs(data):
    from tests import oracle_binding as ob
    _, taps = ob.decode_file(data, taps=True)
    return taps["coeffs"]


def describe(f):
    r = f.reach
    return (f"cells {len(r['cells'])} nz buckets {len(r['nz_buckets'])} lnb {sorted(r['lnb'])} shifts {sorted(r['shifts'])}"
            f" hist {sorted(r['hist'])} full {r['full']} empty {r['empty']} last_k {r['last_k']} wrapped {r['wrapped']}"
            f" max |coeff| {r['max_abs']}")


@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_model(name):
    f, data = model(name)
    want = _CACHE[name][2]
    print(name, describe(f))
    got = oracle_coeffs(data)
    assert np.array_equal(got, f.coeffs), name
    r = f.reach
    if "num_ctx" in want:
        assert f.bcm.num_ctx == want["num_ctx"]
    if "num_lf" in want:
        assert f.bcm.num_lf == want["num_lf"]
        lf_cells = {c % f.bcm.num_lf for c in r["cells"]}
        assert len(lf_cells) >= min(want["num_lf"], 8), lf_cells
    if "qf_buckets" in want:
        assert {(c // f.bcm.num_lf) % 16 for c in r["cells"]} == set(range(16))
    if "hist" in want:
        assert r["hist"] == set(range(want["hist"]))
    if "passes" in want:
        assert len(f.passes) == want["passes"]
    if "wrapped" in want:
        assert r["wrapped"] > 0
    if "orders" in want:
        assert {k[1] // 3 for k in r["orders"]} == set(range(want["orders"]))
    if "edges" in want:
        assert r["max_abs"] == 1 << 25 and 10 in r["lnb"]


def test_matrix_reach():
    """Across the frame set: every (channel, order) cell of the default map, all 36 reachable nonzero buckets, every
    block-count exponent 0..10, shifts 0..3, full and empty blocks and a last coefficient at num_coeffs - 1.
    Bucket 36 (predicted >= 64) cannot be reached: a stored count is shrc(nonzeros, lnb) <= 63 since nonzeros <=
    num_coeffs - num_blocks = 63 * 2^lnb, so every prediction (32, a neighbour or the rounded mean of two) is <= 63."""
    cells, buckets, lnb, shifts = set(), set(), set(), set()
    full = empty = last = 0
    for n in CASES:
        f, _ = model(n)
        if f.bcm.default:
            cells |= f.reach["cells"]
        buckets |= f.reach["nz_buckets"]
        lnb |= f.reach["lnb"]
        shifts |= f.reach["shifts"]
        full += f.reach["full"]
        empty += f.reach["empty"]
        last += f.reach["last_k"]
    assert cells == set(range(39)), sorted(set(range(39)) - cells)
    assert buckets == set(range(36)), sorted(set(range(36)) - buckets)
    assert lnb == set(range(11))
    assert shifts == {0, 1, 2, 3}
    assert full and empty and last


def test_natural_orders_match_golden():
    kat = json.load(open(os.path.join(GOLDEN, "kat.json")))
    assert R.natural_order(0).tolist() == kat["COEFF_ORDER_1X1"]
    assert R.natural_order(4).tolist() == kat["COEFF_ORDER_2X1"]
    for o in range(13):
        assert sorted(R.natural_order(o).tolist()) == list(range(order_size(o)))


# ---------------------------------------------------------------------------------------------------------------
# refusals, each with a valid twin that differs in one token or field
# ---------------------------------------------------------------------------------------------------------------
def _small(chooser_fn, hist=(0,), nh=1, bcm=None, size=64):
    rng = np.random.default_rng(99)
    xb = yb = size // 8
    f = R.Frame(size, size, tile(xb, yb, rng, [0, 4, 5]), lf_field(rng, xb, yb), bcm or R.BlockContextMap(), nh,
                [one_pass(clusters=2)], list(hist))
    return f.decode(chooser_fn)


def _first_block(first):
    """chooser(5), except for the Y channel of the first varblock: first(room) with room = num_coeffs - num_blocks."""
    base = chooser(5)

    def choose(ev):
        if ev["bx"] == 0 and ev["by"] == 0 and ev["c"] == 1:
            return first(ev["num_coeffs"] - ev["num_blocks"])
        return base(ev)
    return choose


def _check_refusal(bad, good, kind):
    import synth
    from jxl_rs_b200 import abi
    assert bad.error == kind and good.error is None
    assert np.array_equal(oracle_coeffs(synth.encode_vardct_tokens(good.spec)), good.coeffs)
    with pytest.raises(abi.JxgError):
        oracle_coeffs(synth.encode_vardct_tokens(bad.spec))


def refusal_pairs():
    def nn(first):
        return lambda: _small(_first_block(first))
    hist = (lambda h: lambda: _small(chooser(3), hist=(0, 1, h, 0), nh=3, size=512))
    return {
        "invalid_num_nonzeros": (nn(lambda room: (room + 1, [])), nn(lambda room: (room, [1] * room)),
                                 "InvalidNumNonZeros"),
        "residual_nonzeros": (nn(lambda room: (2, [0] * (room - 1) + [3])), nn(lambda room: (1, [0] * (room - 1) + [3])),
                              "EndOfBlockResidualNonZeros"),
        "histogram_index": (hist(3), hist(2), "InvalidHistogramIndex"),
    }


@pytest.mark.parametrize("case", ["invalid_num_nonzeros", "residual_nonzeros", "histogram_index"])
def test_refusal_with_twin(case):
    bad, good, kind = refusal_pairs()[case]
    _check_refusal(bad(), good(), kind)


@pytest.mark.parametrize("lf,nq,top,kind", [
    ([[1] * 4, [2] * 12, []], 0, 15, "BlockContextMapSizeTooBig"),   # 5 * 13 = 65 LF contexts
    ([[1] * 3, [2] * 3, [3] * 3], 0, 16, "TooManyBlockContexts"),
    ([[], [], []], 15, 16, "TooManyBlockContexts"),
])
def test_block_context_map_refusals(lf, nq, top, kind):
    """The refused map and its twin (one LF threshold fewer, or the top block context one lower)."""
    import synth
    from jxl_rs_b200 import abi
    qf = list(range(1, nq + 1))

    def bcm_of(lf_, top_):
        n = 1
        for t in lf_:
            n *= len(t) + 1
        cm = [i % (top_ + 1) for i in range(39 * n * (nq + 1))]
        return lf_, cm
    if kind == "BlockContextMapSizeTooBig":
        good_lf = [lf[0][:3], lf[1], lf[2]]
        bad_lf = lf
        tops = (top, top)
    else:
        good_lf = bad_lf = lf
        tops = (top - 1, top)
    g_lf, g_cm = bcm_of(good_lf, tops[0])
    good = _small(chooser(7), bcm=R.BlockContextMap(g_lf, qf, g_cm))
    assert good.error is None
    assert np.array_equal(oracle_coeffs(synth.encode_vardct_tokens(good.spec)), good.coeffs)
    b_lf, b_cm = bcm_of(bad_lf, tops[1])
    with pytest.raises(R.DecodeError) as e:
        R.BlockContextMap(b_lf, qf, b_cm)
    assert e.value.kind == kind
    spec = dict(good.spec)
    spec["bcm"] = {"lf": b_lf, "qf": qf, "map": b_cm}
    with pytest.raises(abi.JxgError):
        oracle_coeffs(synth.encode_vardct_tokens(spec))


# ---------------------------------------------------------------------------------------------------------------
# planted faults
# ---------------------------------------------------------------------------------------------------------------
FAULTS = {
    "no_c_xor": "caught by default_420 (X and Y swap their block contexts)",
    "qf_ge": "caught by qf15 (raw_quant equal to a threshold)",
    "lf_order_xyb": "caught by lf_all64 (Y and B buckets swap places)",
    "pred_no_round": "caught by default_420 (odd sums of the two neighbours)",
    "nz_bucket_63": "caught by ragged_tall_wide or thin (prediction 63 of full neighbours)",
    "freq_k_unshifted": "caught by default_420 (any varblock larger than 8x8)",
    "prev_ge": "caught by default_420 (nonzeros equal to num_coeffs / 16)",
    "perm_inverted": "caught by orders (random permutations)",
    "lehmer_skip0": "caught by orders (permuted orders)",
    "shift_after_prev": "caught by passes11 (values that wrap to 0)",
    "nz_store_floor": "caught by default_420 (counts not a multiple of the block count)",
}


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_planted_fault_is_caught(fault):
    """With the fault, the model's tokens and coefficients, written and decoded by the oracle, differ from what the
    model predicts on at least one frame (the docstring of FAULTS names which)."""
    import synth
    caught = None
    setattr(R.F, fault, True)
    try:
        for name in CASES:
            f, ch, _ = build(name)
            f.decode(ch)
            if f.error is not None:
                caught = name
                break
            try:
                got = oracle_coeffs(synth.encode_vardct_tokens(f.spec))
            except Exception:
                caught = name
                break
            if not np.array_equal(got, f.coeffs):
                caught = name
                break
    finally:
        setattr(R.F, fault, False)
    print(f"fault {fault}: caught by {caught}")
    assert caught is not None, fault
