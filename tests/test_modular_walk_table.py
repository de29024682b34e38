"""Token-level Modular frames aimed at the device's table walk (m_channel_lut in modular_kernels.cu over the table of
modular_batch.cc build_walk_table; specialized_trees.rs:197-372 is the reference's form): hand-written trees whose
channels, once their channel / stream decisions are resolved, split on one property (2..15) or are a single leaf.
They reach every instance of the loop (properties 9, 10 and 13, the single leaf, a property read at run time, with and
without the weighted predictor), the split values at the table's clamp edges and their generic-walk twins just beyond,
neighbours and properties that wrap near +-2^31, channels one to six pixels wide, more than 16 clusters, channel and
stream decisions below a property split, and LZ77 streams.

Here, on the CPU: the oracle decodes each frame to the model's planes and u8 image bit for bit (the oracle has table
walks of its own), each frame reaches what it was built for, and jxg_modular_walk_table routes every channel of every
group stream the way the frame was designed. tests/test_gpu_modular_walk_table.py runs the same frames on the device."""
import collections
import ctypes as C

import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import modular_ref as M
from tests import test_modular_lz77 as L
from tests.test_modular_ref import _bfs, model_planes, oracle_planes

LUT_MIN, LUT_MAX = -1024, 1023  # the table covers property values clamped to [LUT_MIN, LUT_MAX]
NO_WP_PREDS = [0, 1, 2, 3, 4, 5, 7, 8, 9, 10, 11, 12, 13]

# One frame of a case: its designed route per (HF group, channel): a property 2..15, None (a single leaf) or "generic";
# wp_groups: the groups whose tree uses the weighted predictor.
Item = collections.namedtuple("Item", "label frame chooser routes wp_groups")


def sid(g):
    """Stream id of HF group g in a frame of one LF group (1 + 3 * num_lf_groups + 17 + g, mod.rs)."""
    return 21 + g


def leaf(pred, kind=0):
    """kind 0: plain; 1: offset 3; 2: multiplier 2; 3: offset -2 and multiplier 3."""
    return ("leaf", pred, (0, 3, 0, -2)[kind], (0, 0, 1, 0)[kind], (0, 0, 0, 2)[kind])


def leaves(n, preds, start=0):
    """n leaves cycling through `preds` and the four leaf kinds."""
    return [leaf(preds[(start + i) % len(preds)], (start + i + i // len(preds)) % 4) for i in range(n)]


def chain(prop, values, lv):
    """A balanced subtree splitting on `prop` at the increasing `values`, with the leaves `lv` in value order."""
    assert len(lv) == len(values) + 1 and list(values) == sorted(set(values))
    if not values:
        return lv[0]
    m = len(values) // 2
    return ("split", prop, values[m], chain(prop, values[m + 1:], lv[m + 1:]), chain(prop, values[:m], lv[:m + 1]))


def dispatch(prop, subtrees, base=0):
    """Splits on `prop` (0: channel, 1: stream id) choosing subtrees[k] where the property equals base + k."""
    if len(subtrees) == 1:
        return subtrees[0]
    return ("split", prop, base, dispatch(prop, subtrees[1:], base + 1), subtrees[0])


def split_values(prop):
    """Table-walk split values of a property: the table's two ends and values around 0 (y and x are >= 0)."""
    if prop in (2, 3):
        return [LUT_MIN, 2, 5, 60, LUT_MAX - 1]
    if prop in (4, 5):
        return [LUT_MIN, 0, 30, 120, LUT_MAX - 1]
    if prop == 15:
        return [LUT_MIN, -100, -8, 0, 8, 100, LUT_MAX - 1]
    return [LUT_MIN, -20, -1, 0, 3, 40, LUT_MAX - 1]


def prop_tree(prop, preds, start=0):
    """One channel's subtree: a single-property chain, or a single leaf for prop None."""
    if prop is None:
        return leaf(preds[start % len(preds)], start % 4)
    vals = split_values(prop)
    return chain(prop, vals, leaves(len(vals) + 1, preds, start))


def target_chooser(seed, targets, p_target, p_small=0.1):
    """Residuals that put a share `p_target` of the pixels exactly on values drawn from `targets` (the decoded value
    wraps to the target), the rest toward picture_chooser's smooth picture."""
    rng = np.random.default_rng(seed)
    pic = M.picture_chooser(seed + 1, p_small=p_small)

    def choose(guess, mul, x, y, c):
        if rng.random() < p_target:
            t = int(targets[int(rng.integers(len(targets)))])
            return M.wrap32(t - guess) if mul == 1 else M.clamp_dec((t - guess) // mul, mul)
        return pic(guess, mul, x, y, c)
    return choose


# ---------------------------------------------------------------------------------------------------------------------
# The cases
# ---------------------------------------------------------------------------------------------------------------------
def _each_property():
    """300 x 280 (3 x 3 groups of 128): the global tree dispatches on the stream id, then the channel, to one
    single-property chain (or single leaf) per channel of groups 0..6, without the weighted predictor; groups 7 and 8
    have local trees that use it, on property 15, on properties 4, 9 and 13 and on a single leaf."""
    slots = [2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, None, 9, 10, 13, 8, None, 14, 12]  # groups 0..6, channels 0..2
    routes = {(g, c): slots[g * 3 + c] for g in range(7) for c in range(3)}
    per_stream = [dispatch(0, [prop_tree(slots[g * 3 + c], NO_WP_PREDS, 5 * g + c) for c in range(3)]) for g in range(7)]
    per_stream += [leaf(1), leaf(2)]  # groups 7 and 8 read their local trees
    wp_preds = [6, 6, 1, 13, 6, 5, 6, 12]
    local = {7: [15, 4, None], 8: [15, 9, 13]}
    groups = {}
    for g, props in local.items():
        groups[g] = {"tree": _bfs(dispatch(0, [prop_tree(p, wp_preds, 3 * c + g) for c, p in enumerate(props)])),
                     "wp": (12, 9, 5, 7, 9, 3, 2, 11, 13, 12, 10) if g == 7 else None}
        routes.update({(g, c): p for c, p in enumerate(props)})
    frame = M.Frame(300, 280, _bfs(dispatch(1, per_stream, sid(0))), group_shift=0, groups=groups)
    return [Item("each_property", frame, M.picture_chooser(44, p_small=0.15, p_huge=0.03), routes, {7, 8})]


EDGE_TARGETS = [-1026, -1025, -1024, -1023, -1022, 1021, 1022, 1023, 1024, 1025, -1, 0, 1, 2, M.I32_MIN, M.I32_MIN + 1,
                M.I32_MAX, 5000, -5000, 1 << 20, -(1 << 20)]


def _clamp_edges():
    """Two 200 x 140 frames: in one, every channel splits at LUT_MIN and LUT_MAX - 1 (properties 7 = W, 6 = N and
    5 = |W|, table walk); in its twin, channel 0 splits at LUT_MIN - 1, channel 1 at LUT_MAX and channel 2 at both, so
    that each limit alone sends the channel to the generic walk. Pixels sit on both sides of every split value."""
    def tree(lo, hi):
        return _bfs(dispatch(0, [chain(7, [lo[0], 0, hi[0]], leaves(4, NO_WP_PREDS, 0)),
                                 chain(6, [lo[1], 0, hi[1]], leaves(4, NO_WP_PREDS, 4)),
                                 chain(5, [lo[2], 1, hi[2]], leaves(4, NO_WP_PREDS, 8))]))
    a, b = LUT_MIN, LUT_MAX - 1
    table = M.Frame(200, 140, tree((a, a, a), (b, b, b)), group_shift=0)
    twin = M.Frame(200, 140, tree((a - 1, a, a - 1), (b, b + 1, b + 1)), group_shift=0)
    return [Item("clamp_edges_table", table, target_chooser(51, EDGE_TARGETS, 0.6), {(g, c): 7 - c for g in range(4)
                                                                                     for c in range(3)}, set()),
            Item("clamp_edges_generic", twin, target_chooser(51, EDGE_TARGETS, 0.6),
                 {(g, c): "generic" for g in range(4) for c in range(3)}, set())]


WRAP_TARGETS = [M.I32_MIN, M.I32_MIN + 1, M.I32_MIN + 2, M.I32_MAX, M.I32_MAX - 1, M.I32_MAX - 2, -(1 << 30), 1 << 30,
                -1, 0, 1]
WRAP_PREDS = [3, 4, 5, 10, 11, 12, 13]


def _wrapped_neighbours():
    """260 x 140 (3 x 2 groups): pixels at and near i32::MIN and i32::MAX next to small ones, under chains on properties
    4, 5 and 8..14 (two channels each) whose leaves use the predictors that average or compare neighbours, two of them
    with offsets at the i32 ends."""
    props = [4, 5, 8, 9, 10, 11, 12, 13, 14] * 2
    wide = [("leaf", 5, M.I32_MAX, 0, 0), ("leaf", 13, M.I32_MIN, 0, 0)]
    per_stream = []
    for g in range(6):
        subs = []
        for c in range(3):
            p = props[g * 3 + c]
            vals = [LUT_MIN, -1, 0, 1, LUT_MAX - 1]
            lv = leaves(len(vals) + 1, WRAP_PREDS, g * 3 + c)
            if (g * 3 + c) % 4 == 0:
                lv[-1] = wide[(g + c) % 2]
            subs.append(chain(p, vals, lv))
        per_stream.append(dispatch(0, subs))
    frame = M.Frame(260, 140, _bfs(dispatch(1, per_stream, sid(0))), group_shift=0)
    routes = {(g, c): props[g * 3 + c] for g in range(6) for c in range(3)}
    return [Item("wrapped_neighbours", frame, target_chooser(61, WRAP_TARGETS, 0.5), routes, set())]


def _narrow_channels():
    """Grey frames of (128 + w) x (128 + h) for w in 1..6 and h in 1..3: their right groups are w pixels wide (no,
    one or two interior pixels per row), the bottom ones h rows high, the corner one w x h. Property 8 (W minus the
    previous pixel's gradient) on the narrow groups carries across the seam between the edge and interior pixels;
    their leaves use AverageAll (its top-right-right neighbour) and the left-left neighbour."""
    out = []
    for w in range(1, 7):
        for h in range(1, 4):
            per_stream = [chain(14, [LUT_MIN, -2, 0, 2, LUT_MAX - 1], leaves(6, [13, 9, 5, 1, 13, 12])),
                          chain(8, [LUT_MIN, -3, 0, 3, 30, LUT_MAX - 1], leaves(7, [13, 9, 13, 5, 13, 1, 11], w)),
                          chain(13, [LUT_MIN, -4, 0, 4, LUT_MAX - 1], leaves(6, [13, 3, 9, 13, 2, 7], h)),
                          chain(8, [-3, 0, 3], leaves(4, [13, 9, 13, 12], w + h))]
            frame = M.Frame(128 + w, 128 + h, _bfs(dispatch(1, per_stream, sid(0))), group_shift=0, grey=True)
            out.append(Item(f"narrow_{w}x{h}", frame, M.picture_chooser(70 + 3 * w + h, p_small=0.4, p_huge=0.01),
                            {(0, 0): 14, (1, 0): 8, (2, 0): 13, (3, 0): 8}, set()))
    return out


MANY = sorted({int(round(v)) for v in np.linspace(LUT_MIN, LUT_MAX - 1, 254)})


def _many_clusters():
    """200 x 140 with prefix codes: one chain of 254 splits on property 7 (W) over the whole table, 255 leaves, so
    cluster ids (one per leaf) run up to 254, the largest a context map of 255 leaf contexts holds."""
    assert len(MANY) == 254
    tree = _bfs(chain(7, MANY, leaves(255, NO_WP_PREDS)))
    targets = list(range(LUT_MIN - 40, LUT_MAX + 40))
    frame = M.Frame(200, 140, tree, group_shift=0, prefix=True)
    return [Item("many_clusters", frame, target_chooser(81, targets, 0.7), {(g, c): 7 for g in range(4)
                                                                            for c in range(3)}, set())]


def _inner_static():
    """300 x 140 (3 x 2 groups): the global tree splits on property 9 first and decides on the channel (left) or the
    stream id (right) below it; groups 1 and 4 have local trees that split on property 10 first and then on the stream
    id and the channel. Each (channel, stream) then has a table of its own, which the walk cache must key by both."""
    right = dispatch(1, [chain(9, [-40, -5], leaves(3, NO_WP_PREDS, 2 * g)) for g in range(6)], sid(0))
    left = dispatch(0, [chain(9, [5, 40], leaves(3, NO_WP_PREDS, 3 + c)) for c in range(2)] + [leaf(13, 3)])
    gtree = _bfs(("split", 9, 0, left, right))
    groups = {}
    for g in (1, 4):
        lo = dispatch(0, [chain(10, [-30, -2], leaves(3, [13, 5, 1, 11], c + g)) for c in range(3)])
        hi = dispatch(1, [chain(10, [4, 30], leaves(3, [12, 9, 3, 4], g)), leaf(0, 1)], sid(g))
        groups[g] = {"tree": _bfs(("split", 10, 1, hi, lo))}
    frame = M.Frame(300, 140, gtree, group_shift=0, groups=groups)
    routes = {(g, c): 10 if g in groups else 9 for g in range(6) for c in range(3)}
    return [Item("inner_static", frame, M.picture_chooser(91, p_small=0.3, p_huge=0.02), routes, set())]


BUILDERS = {"each_property": _each_property, "clamp_edges": _clamp_edges, "wrapped_neighbours": _wrapped_neighbours,
            "narrow_channels": _narrow_channels, "many_clusters": _many_clusters, "inner_static": _inner_static}
CASES = list(BUILDERS)
LZ77_CASES = {"each_property": 2, "inner_static": 1}  # case -> LZ77 mode of its copy (test_modular_lz77.token_frame)
_CACHE = {}


def items(name):
    """The case's frames, decoded by the model, each with its written file: [(Item, bytes)]."""
    if name not in _CACHE:
        import synth
        out = []
        for it in BUILDERS[name]():
            it.frame.decode(it.chooser)
            out.append((it, synth.encode_modular_tokens(it.frame.spec)))
        _CACHE[name] = out
    return _CACHE[name]


def lz77_items(name):
    """The case's frames written with LZ77 copies: [(Item, bytes, census)]."""
    import synth
    key = ("lz77", name)
    if key not in _CACHE:
        out = []
        for it, _ in items(name):
            spec = dict(it.frame.spec)
            spec["lz77"] = {"mode": LZ77_CASES[name], "multipliers": L.multipliers(it.frame)}
            data = synth.encode_modular_tokens(spec)
            out.append((it, data, synth.lz77_census()))
        _CACHE[key] = out
    return _CACHE[key]


def hf_rects(frame):
    """(group, channel) of every non-empty group-stream rect."""
    nc = 1 if frame.grey else 3
    _, rects, _ = M.section_layout(frame.w, frame.h, frame.group_shift, nc)
    return {(g, c) for g, r in enumerate(rects) if r[2] and r[3] for c in range(nc)}


def expected_walk_stats(its):
    """What ModularBatch.walk_stats() must count for frames `its`, from their designed routes."""
    st = {"generic": 0, "single_leaf": 0, "by_property": collections.Counter(), "table_wp": 0}
    for it in its:
        for (g, _), r in it.routes.items():
            if r == "generic":
                st["generic"] += 1
                continue
            if r is None:
                st["single_leaf"] += 1
            else:
                st["by_property"][r] += 1
            st["table_wp"] += g in it.wp_groups
    st["by_property"] = dict(st["by_property"])
    return st


def walk_table(tree, channel, stream_id):
    """jxg_modular_walk_table for a BFS tree of the model (one context per leaf, context = cluster): (1, property or
    0xff, table) or (0, None, None)."""
    nodes, _ = M.link_tree(tree)
    flat = []
    for n in nodes:
        if n[0] == "split":
            flat += [n[1], n[2], n[3], n[4], 0]
        else:
            flat += [-1, n[2], n[1], M.wrap32(n[3]), n[4]]
    n_ctx = sum(n[0] == "leaf" for n in nodes)
    arr = np.array(flat, np.int32)
    cmap = np.arange(n_ctx, dtype=np.uint8)
    lut = np.zeros(2048, np.uint32)
    prop = C.c_uint32(0)
    lib = abi.load_library()
    r = lib.jxg_modular_walk_table(arr.ctypes.data_as(C.POINTER(C.c_int32)), len(nodes),
                                   cmap.ctypes.data_as(C.POINTER(C.c_uint8)), n_ctx, channel, stream_id,
                                   lut.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(prop))
    assert r in (0, 1), r
    return (1, prop.value, lut) if r else (0, None, None)


# ---------------------------------------------------------------------------------------------------------------------
# What each case must reach, so that a change of seed cannot quietly empty it
# ---------------------------------------------------------------------------------------------------------------------
def _both_sides(cov, prop, val):
    return (prop, val, False) in cov.split_sides and (prop, val, True) in cov.split_sides


def _check_reach(name, its):
    cov = M.Coverage()
    for it in its:
        cov.merge(it.frame.cov)
    if name == "each_property":
        assert cov.predictors == set(range(14)), sorted(cov.predictors)
        for p in range(2, 16):  # every property's split near 0 goes both ways
            near = [v for v in split_values(p) if -30 <= v <= 60]
            assert any(_both_sides(cov, p, v) for v in near), p
        for p in range(4, 16):  # and values beyond the table at both ends, on the properties that can have them
            if p != 15:
                assert _both_sides(cov, p, LUT_MAX - 1), p
        assert cov.offset_leaves > 100 and cov.mul_leaves > 100
    elif name == "clamp_edges":  # both sides of every split, with the property exactly at the split value and one above
        for p, val in {(n[1], n[2]) for it in its for n in it.frame.tree if n[0] == "split" and n[1] >= 2}:
            if p == 5 and val < 0:  # |W| < 0 only for W = i32::MIN (wrapping_abs)
                assert (5, val, False) in cov.split_sides, val
                continue
            assert _both_sides(cov, p, val), (p, val)
            assert (p, val, 0) in cov.split_edges and (p, val, 1) in cov.split_edges, (p, val)
        for p in (6, 7):
            assert cov.prop_range[p][0] < -(1 << 20) and cov.prop_range[p][1] > (1 << 20)
        assert cov.prop_range[5][0] == M.I32_MIN
    elif name == "wrapped_neighbours":
        assert cov.predictors >= set(WRAP_PREDS)
        assert cov.wrapped_props == set(range(8, 15)), sorted(cov.wrapped_props)
        assert cov.prop_range[4][0] == M.I32_MIN and cov.prop_range[5][0] == M.I32_MIN
        assert cov.wrapped > 1000 and cov.offset_leaves > 100
        for p in (4, 5, 8, 9, 10, 11, 12, 13, 14):
            assert _both_sides(cov, p, 0) and _both_sides(cov, p, LUT_MAX - 1), p
    elif name == "narrow_channels":
        assert _both_sides(cov, 8, 0) and _both_sides(cov, 8, 3) and 13 in cov.predictors and 9 in cov.predictors
    elif name == "many_clusters":
        missing = [v for v in MANY if not _both_sides(cov, 7, v)]  # every split both ways: all 255 leaves reached
        assert not missing, missing
    elif name == "inner_static":
        for p, v in ((9, 0), (9, 5), (9, 40), (9, -5), (9, -40), (10, 1), (10, -2), (10, 4)):
            assert _both_sides(cov, p, v), (p, v)


# ---------------------------------------------------------------------------------------------------------------------
# Tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_model_equals_oracle(name):
    its = items(name)
    for it, data in its:
        out, planes = oracle_planes(data)
        assert np.array_equal(planes.reshape(-1), model_planes(it.frame).reshape(-1).astype(np.int32)), it.label
        assert np.array_equal(out, it.frame.u8), it.label
    _check_reach(name, [it for it, _ in its])


@pytest.mark.parametrize("name", CASES)
def test_host_routes_are_the_designed_ones(name):
    """Every non-empty group-stream rect has a designed route, and jxg_modular_walk_table (the batch's
    build_walk_table) gives that route for its channel and stream id: the table over the designed property, the
    single-leaf table, or the generic walk."""
    for it, _ in items(name):
        assert set(it.routes) == hf_rects(it.frame), it.label
        for (g, c), want in it.routes.items():
            tree = it.frame.groups.get(g, {}).get("tree") or it.frame.tree
            ok, prop, _ = walk_table(tree, c, sid(g))
            if want == "generic":
                assert ok == 0, (it.label, g, c)
            else:
                assert ok == 1 and prop == (0xFF if want is None else want), (it.label, g, c, prop)


def test_cases_reach_every_table_instance():
    """Between them the designed routes take each instance of m_channel_lut: properties 9, 10 and 13, the single leaf
    and a property read at run time, without the weighted predictor, and with it on property 15, on another property
    and on a single leaf; and the generic walk for the clamp-edge twins."""
    no_wp, wp = set(), set()
    generic = 0
    for name in CASES:
        for it, _ in items(name):
            for (g, _), r in it.routes.items():
                if r == "generic":
                    generic += 1
                else:
                    (wp if g in it.wp_groups else no_wp).add(r)
    assert {9, 10, 13, None} <= no_wp and no_wp - {9, 10, 13, None}, no_wp
    assert {15, None} <= wp and wp - {15, None}, wp
    assert generic == 12


@pytest.mark.parametrize("name", sorted(LZ77_CASES))
def test_lz77_frames_equal_the_model(name):
    """The same frames with LZ77 copies in their group streams (the LZ = true instances of the loop)."""
    for it, data, census in lz77_items(name):
        out, planes = oracle_planes(data)
        assert np.array_equal(planes.reshape(-1), model_planes(it.frame).reshape(-1).astype(np.int32)), it.label
        assert np.array_equal(out, it.frame.u8)
        assert census["copies"] > 100, census
