"""The Modular decode against tests/modular_ref.py, a plain-integer restatement of the reference, on token-level frames
(synth.encode_modular_tokens): the model decodes forward and chooses every symbol, the writer only serialises, and the
oracle (the front-end's decoder, csrc/host/modular.cc) must return the model's i32 planes and u8 image bit for bit.
Also the tree and transform refusals of the reference, and planted faults in the model. No GPU."""
import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import modular_ref as M

ALL_PROPS = list(range(24)) + [24, 25, 26, 27]
# RCT types 0..41 spread over the local RCT lists of nine groups, five per group
LOCAL_RCT = {g: [(0, t) for t in range(g * 5, min(g * 5 + 5, 42))] for g in range(9)}


def _wp(rng):
    return tuple(int(v) for v in rng.integers(0, 32, 7)) + tuple(int(v) for v in rng.integers(0, 16, 4))


def _case(name):
    """(Frame, chooser) of one matrix case; trees and headers are random but fixed per case name."""
    rng = np.random.default_rng(sum(map(ord, name)))
    tree = lambda depth=5, props=ALL_PROPS, **kw: M.random_tree(rng, depth, props, **kw)  # noqa: E731
    pic = M.picture_chooser(sum(map(ord, name)) + 1)
    if name == "1x1":
        return M.Frame(1, 1, tree(2), group_shift=0, orientation=2), pic
    if name == "one_row":
        return M.Frame(300, 1, tree(), group_shift=0, orientation=4, hybrid=(2, 1, 1)), pic
    if name == "two_columns":
        return M.Frame(2, 300, tree(), group_shift=0, orientation=7, prefix=True), pic
    if name == "edge_rects_128":  # groups of 3 x 2 and 2 x 2 pixels at the right and bottom edges
        return M.Frame(259, 130, tree(6), group_shift=0, orientation=5, global_rct=[(0, 6)]), pic
    if name == "groups_256":
        return M.Frame(300, 270, tree(6), group_shift=1, orientation=8, hybrid=(0, 0, 0), global_rct=[(0, 13)]), pic
    if name == "global_rct_0_20":
        return M.Frame(140, 130, tree(), group_shift=0, global_rct=[(0, t) for t in range(21)]), \
            M.picture_chooser(5, p_small=0.1, p_huge=0.05)
    if name == "global_rct_21_41":
        return M.Frame(140, 130, tree(), group_shift=0, prefix=True, orientation=3,
                       global_rct=[(0, t) for t in range(21, 42)]), M.picture_chooser(6, p_small=0.1, p_huge=0.05)
    if name == "local_rct_wp_local_trees":  # nine groups: own WeightedHeaders, local RCTs, local trees in four
        groups = {g: {"wp": _wp(rng), "rct": LOCAL_RCT[g],
                      "tree": tree(4, [15, 0, 1, 9, 10], leaf_preds=[6, 6, 5, 13]) if g % 2 else None} for g in range(9)}
        return M.Frame(300, 260, tree(5, [15, 0, 2, 3, 6], leaf_preds=[6, 6, 1, 4]), group_shift=0, orientation=6,
                       groups=groups, global_wp=_wp(rng)), M.picture_chooser(7, p_small=0.2, p_huge=0.02)
    if name == "wp_default":
        return M.Frame(200, 150, tree(5, [15, 0, 8, 9, 14], leaf_preds=[6, 6, 6, 3]), group_shift=0), pic
    if name == "wp_random_extreme":
        return M.Frame(140, 140, tree(4, [15, 0, 11, 12], leaf_preds=[6, 6, 6, 7, 9]), group_shift=0,
                       groups={g: {"wp": _wp(rng)} for g in range(4)}, global_wp=_wp(rng)), \
            M.picture_chooser(8, p_small=0.1, p_huge=0.3)
    if name == "wide_leaves_wrap":
        return M.Frame(150, 140, tree(6, big_values=True, wide_leaves=True), group_shift=0, prefix=True), \
            M.picture_chooser(9, p_small=0.2, p_huge=0.2)
    if name == "reference_slots":
        lf = lambda p: ("leaf", p, 0, 0, 0)  # noqa: E731
        t = _bfs(("split", 0, 1, ("split", 21, 120, ("split", 23, 0, lf(1), lf(2)), ("split", 17, 60, lf(5), lf(7))),
                  ("split", 19, 0, ("split", 16, 30, lf(9), lf(3)), ("split", 20, 90, lf(11), ("split", 24, 0, lf(0), lf(12))))))
        return M.Frame(130, 130, t, group_shift=0, global_rct=[(0, 40)]), M.picture_chooser(10, p_small=0.3)
    if name == "explicit_splits":  # |W| (5) and the first reference slot's |gradient residual| (18), hand-placed
        lf = lambda p: ("leaf", p, 0, 0, 0)  # noqa: E731
        t = _bfs(("split", 0, 0, ("split", 18, 6, lf(1), lf(2)), ("split", 5, 100, lf(5), lf(3))))
        return M.Frame(80, 60, t, group_shift=0), M.picture_chooser(11, p_small=0.3)
    if name == "palette_one_group":  # palette meta channel and index channel both in the global section
        return M.Frame(100, 90, tree(4, [0, 1, 3, 6, 7]), group_shift=0, palette=(37, M.index_chooser(12, 37)),
                       orientation=4), pic
    if name == "palette_groups":  # index channel over the HF groups, with local trees and WeightedHeaders
        return M.Frame(270, 140, tree(4, [0, 2, 5, 15], leaf_preds=[0, 1, 5, 6]), group_shift=0, prefix=True,
                       palette=(300, M.index_chooser(13, 300)),
                       groups={1: {"tree": tree(3, [3, 4, 10]), "wp": _wp(rng)}, 4: {"wp": _wp(rng)}}), pic
    if name == "grey":
        return M.Frame(260, 140, tree(5, [0, 1, 2, 3, 4, 5, 6, 7, 15]), group_shift=0, grey=True, orientation=5), pic
    if name == "grey_single_group":
        return M.Frame(100, 60, tree(4, [3, 8, 13, 14]), group_shift=1, grey=True, orientation=2, prefix=True), pic
    raise KeyError(name)


CASES = ["1x1", "one_row", "two_columns", "edge_rects_128", "groups_256", "global_rct_0_20", "global_rct_21_41",
         "local_rct_wp_local_trees", "wp_default", "wp_random_extreme", "wide_leaves_wrap", "reference_slots", "explicit_splits",
         "palette_one_group", "palette_groups", "grey",
         "grey_single_group"]
_CACHE = {}


def model(name):
    """Model result and the written file of one case, cached per module (the model is per-pixel Python)."""
    if name not in _CACHE:
        import synth
        frame, chooser = _case(name)
        frame.decode(chooser)
        _CACHE[name] = (frame, synth.encode_modular_tokens(frame.spec))
    return _CACHE[name]


def oracle_planes(data):
    from tests import oracle_binding as ob
    out, planes = ob.decode_modular_file(data, planes=True)
    return out, planes


def model_planes(frame):
    p = frame.planes
    if p.shape[0] == 1:
        p = np.repeat(p, 3, axis=0)
    return p  # as coded, like the oracle's planes (which it allocates as (3, w, h) of the display size for 5..8)


# What each case must reach, so that a change of seed cannot quietly empty it: (predictors at least, properties split
# both ways at least, properties that must be split both ways, other required features)
REACH = {
    "1x1": (1, 0, set(), set()),
    "one_row": (2, 1, set(), set()),
    "two_columns": (3, 3, set(), {"offset", "mul"}),
    "edge_rects_128": (6, 8, {15, 22}, {"offset", "refs"}),
    "groups_256": (2, 1, set(), set()),
    "global_rct_0_20": (4, 4, set(), {"wrapped"}),
    "global_rct_21_41": (1, 0, set(), {"wrapped"}),
    "local_rct_wp_local_trees": (4, 4, {0, 1, 15}, {"offset", "mul", "wrapped"}),
    "wp_default": (2, 3, {0, 15}, {"offset"}),
    "wp_random_extreme": (3, 3, {15}, {"offset", "wrapped", "wrapped_props"}),
    "wide_leaves_wrap": (8, 12, set(), {"offset", "mul", "wrapped", "wrapped_props", "refs"}),
    "reference_slots": (6, 6, {0, 16, 17, 19, 21, 23}, {"refs"}),
    "explicit_splits": (4, 3, {0, 5, 18}, set()),
    "palette_one_group": (2, 1, set(), {"palette"}),
    "palette_groups": (2, 1, set(), {"palette"}),
    "grey": (3, 2, set(), {"offset", "mul"}),
    "grey_single_group": (2, 1, set(), set()),
}


def _both(cov):
    return {p for p, b in cov.branches if (p, not b) in cov.branches}


@pytest.mark.parametrize("name", CASES)
def test_model_equals_oracle(name):
    frame, data = model(name)
    out, planes = oracle_planes(data)
    assert np.array_equal(planes.reshape(-1), model_planes(frame).reshape(-1).astype(np.int32))
    assert np.array_equal(out, frame.u8)
    n_pred, n_both, props, feats = REACH[name]
    cov = frame.cov
    assert len(cov.predictors) >= n_pred and len(_both(cov)) >= n_both and props <= _both(cov), (
        sorted(cov.predictors), sorted(_both(cov)))
    reached = {"offset": cov.offset_leaves > 0, "mul": cov.mul_leaves > 0, "wrapped": cov.wrapped > 0,
               "wrapped_props": bool(cov.wrapped_props), "refs": cov.ref_slots == {0, 1},
               "palette": cov.palette == {"negative", "explicit", "small_cube", "large_cube", "beyond_cube"}}
    assert all(reached[f] for f in feats), {f: reached[f] for f in feats}


def test_matrix_reaches_every_feature():
    """What the case matrix reached, over all cases: every predictor, both branches of properties 0..23 and splits on
    the reference slots beyond (24..27 read 0 with three channels: a pixel has at most two earlier channels of its
    size), offset and multiplier leaves, wrapped make_pixel results, all 42 RCT types as global and as group-local
    transforms, both entropy codings, three hybrid-uint configurations, group sizes 128 and 256, orientations 1..8 and
    grey, every kind of palette index, and wrapped values of properties 8..14."""
    cov = M.Coverage()
    for name in CASES:
        cov.merge(model(name)[0].cov)
    frames = [model(n)[0] for n in CASES]
    assert cov.predictors == set(range(14))
    missing = [(p, b) for p in range(24) for b in (False, True) if (p, b) not in cov.branches]
    assert not missing, missing
    assert {p for p, _ in cov.branches} >= {24, 27}
    assert cov.ref_slots == {0, 1}
    assert cov.offset_leaves > 100 and cov.mul_leaves > 100 and cov.wrapped > 100
    assert cov.wrapped_props == set(range(8, 15))
    assert cov.palette == {"negative", "explicit", "small_cube", "large_cube", "beyond_cube"}
    assert cov.rct == set(range(42)) and cov.local_rct == set(range(42))
    assert {f.prefix for f in frames} == {False, True}
    assert {f.hybrid for f in frames} >= {(4, 2, 0), (2, 1, 1), (0, 0, 0)}
    assert {f.group_shift for f in frames} == {0, 1}
    assert {f.orientation for f in frames} == set(range(1, 9))
    assert any(f.grey for f in frames)


# ---------------------------------------------------------------------------------------------------------------------
# Refusals
# ---------------------------------------------------------------------------------------------------------------------
def _chain(n, prop=3):
    """A tree of height n: splits on `prop` at -1, -2, ..., each with a leaf on its left and the next split on its
    right; every pixel (x >= 0) takes the first left branch, so the model walks it in one step."""
    out = []
    for k in range(n):
        out += [("split", prop, -1 - k), ("leaf", 5, 0, 0, 0)]
    return out + [("leaf", 0, 0, 0, 0)]


def _bfs(root):
    out, q = [], [root]
    while q:
        n = q.pop(0)
        out.append(n[:3] if n[0] == "split" else n)
        if n[0] == "split":
            q += [n[3], n[4]]
    return out


L = ("leaf", 5, 0, 0, 0)
REFUSALS = [
    # (name, refused tree, its valid boundary twin)
    ("child_contradicts_parent", _bfs(("split", 6, 10, ("split", 6, 5, L, L), L)),
     _bfs(("split", 6, 10, ("split", 6, 11, L, L), L))),
    ("right_child_at_upper_bound", _bfs(("split", 6, 10, L, ("split", 6, 10, L, L))),
     _bfs(("split", 6, 10, L, ("split", 6, 9, L, L)))),
    ("left_child_below_lower_bound", _bfs(("split", 7, -3, ("split", 7, -3, L, L), L)),
     _bfs(("split", 7, -3, ("split", 7, -2, L, L), L))),
    ("root_at_i32_max", [("split", 6, M.I32_MAX), L, L], [("split", 6, M.I32_MAX - 1), L, L]),
    ("height_2049", _chain(2049), _chain(2048)),
    ("mul_log_31", [("leaf", 5, 0, 31, 0)], [("leaf", 5, 0, 30, 2)]),
    ("multiplier_above_u32", [("leaf", 5, 0, 30, 3)], [("leaf", 5, 0, 0, 0xFFFFFFFE)]),
    ("predictor_14", [("leaf", 14, 0, 0, 0)], [("leaf", 13, 0, 0, 0)]),
    ("property_256", [("split", 256, 0), L, L], [("split", 255, 0), L, L]),
]


def _refusal_frame(tree, check, **kw):
    return M.Frame(130, 130, tree, group_shift=0, check=check, **kw).decode(M.picture_chooser(3))


def _assert_refused(data):
    from tests import oracle_binding as ob
    with pytest.raises(abi.JxgError):
        ob.decode_modular_file(data)


@pytest.mark.parametrize("name,bad,good", REFUSALS, ids=[r[0] for r in REFUSALS])
@pytest.mark.parametrize("where", ["global", "local"])
def test_tree_refusals(name, bad, good, where):
    """Each refused tree raises in the model (tree.rs:284-353 / validate_tree) and makes the oracle fail, as the
    global tree and as one group's local tree; its boundary twin decodes and matches the model. The VarDCT front-end
    reads its LF, HF-metadata and quant-table trees with the same ModularTree::read (frame.cc), so these refusals
    cover VarDCT frames too."""
    import synth
    with pytest.raises(M.TreeRefused):
        M.link_tree(bad)
    base = [("leaf", 5, 0, 0, 0)]
    for tree, ok in ((bad, False), (good, True)):
        if where == "global":
            f = _refusal_frame(tree, ok)
        else:
            f = _refusal_frame(base, ok, groups={0: {"tree": tree}})
        data = synth.encode_modular_tokens(f.spec)
        if ok:
            out, planes = oracle_planes(data)
            assert np.array_equal(planes.astype(np.int64), f.planes) and np.array_equal(out, f.u8)
        else:
            _assert_refused(data)


PALETTE_REFUSALS = [
    # (name, frame kwargs): check_equal_channels (meta_apply.rs:188) and RCT after the palette leaves two channels
    ("palette_four_channels", {"palette": (20, M.index_chooser(1, 20), 0, 4)}),
    ("palette_begin_1", {"palette": (20, M.index_chooser(1, 20), 1, 3)}),
    ("palette_three_on_grey", {"palette": (20, M.index_chooser(1, 20), 0, 3), "grey": True}),
    ("rct_after_palette", {"palette": (20, M.index_chooser(1, 20)), "global_rct": [(0, 6)]}),
]


@pytest.mark.parametrize("name,kw", PALETTE_REFUSALS, ids=[r[0] for r in PALETTE_REFUSALS])
def test_palette_range_refusals(name, kw):
    import synth
    with pytest.raises(M.TreeRefused):
        _refusal_frame([("leaf", 5, 0, 0, 0)], True, **kw)
    f = _refusal_frame([("leaf", 5, 0, 0, 0)], False, **kw)
    _assert_refused(synth.encode_modular_tokens(f.spec))


def _cpp_table(path, name):
    import os
    import re
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), path)).read()
    body = src[src.index(name):]
    body = body[body.index("= {") + 3:body.index("};")]
    return [[int(v) for v in m] for m in re.findall(r"\{\s*(-?\d+),\s*(-?\d+),\s*(-?\d+)\s*\}", body)]


def test_delta_palette_copies_equal_the_fixture():
    """The 72-entry delta table (tests/golden/modular_delta_palette.json, taken from the reference) against the copies
    the device kernel and the host decoder carry."""
    want = M.DELTA_PALETTE
    assert len(want) == 72
    assert _cpp_table("jxl_rs_b200/csrc/cuda/modular_kernels.cu", "c_palette_delta") == want
    assert _cpp_table("jxl_rs_b200/csrc/host/modular.cc", "kDelta[72][3]") == want


@pytest.mark.parametrize("rct,grey,local", [((0, 42), False, False), ((0, 42), False, True), ((1, 6), False, False),
                                            ((1, 6), False, True), ((0, 6), True, False)])
def test_transform_refusals(rct, grey, local):
    """RCT type 42 (headers/modular.rs: rct_type < 42) and an RCT beyond the channels (meta_apply.rs:62
    check_equal_channels), global and group-local, and on a grey frame."""
    import synth
    kw = {"groups": {2: {"rct": [rct]}}} if local else {"global_rct": [rct]}
    with pytest.raises(M.TreeRefused):
        _refusal_frame([("leaf", 5, 0, 0, 0)], True, grey=grey, **kw)
    f = _refusal_frame([("leaf", 5, 0, 0, 0)], False, grey=grey, **kw)
    _assert_refused(synth.encode_modular_tokens(f.spec))


# ---------------------------------------------------------------------------------------------------------------------
# Planted faults
# ---------------------------------------------------------------------------------------------------------------------
def _fault_caught(frame, chooser):
    """A model with a planted fault writes a frame whose symbols and pixels follow the fault; the oracle must then
    either refuse the stream or decode pixels that differ from the faulty model's."""
    import synth
    from tests import oracle_binding as ob
    frame.decode(chooser)
    data = synth.encode_modular_tokens(frame.spec)
    try:
        out, planes = ob.decode_modular_file(data, planes=True)
    except abi.JxgError:
        return True
    return not np.array_equal(planes.reshape(-1), model_planes(frame).reshape(-1).astype(np.int32))


FAULTS = [
    # (fault, frame factory, chooser): each docstring line says whether the round trip of the writer
    # (test_cpu_modular.test_lossless_roundtrip) would have caught the same fault in the front-end
    ("prop9_carry",  # round trip: no (no synthetic tree splits on property 8)
     lambda: M.Frame(120, 40, [("split", 8, 0), ("leaf", 5, 0, 0, 0), ("leaf", 1, 0, 0, 0)]), M.picture_chooser(1, p_small=0.5)),
    ("select_tie_west",  # round trip: yes (tree kind 1 has a Select leaf, and the writer predicts on its own)
     lambda: M.Frame(120, 40, [("leaf", 4, 0, 0, 0)]), M.picture_chooser(2, p_small=1.0)),
    ("avgall_trr_top",  # round trip: no (the writer maps AverageAll to the gradient)
     lambda: M.Frame(120, 40, [("leaf", 13, 0, 0, 0)]), M.picture_chooser(3, p_small=0.5)),
    ("wp_saturate",  # round trip: no (the writer tokenises with the front-end's own WpState)
     lambda: M.Frame(120, 60, [("leaf", 6, 0, 0, 0)]), M.picture_chooser(4, p_huge=0.5)),
    ("rct_gbr_brg_swapped",  # round trip: no (the writer only uses RCT type 6)
     lambda: M.Frame(120, 40, [("leaf", 5, 0, 0, 0)], global_rct=[(0, 7 + 3)]), M.picture_chooser(5)),
    ("refs_farthest_first",  # round trip: yes for channel 2 of tree kind 3, which splits on property 17
     lambda: M.Frame(120, 40, [("split", 17, 100), ("leaf", 1, 0, 0, 0), ("leaf", 2, 0, 0, 0)]), M.picture_chooser(6, p_small=0.3)),
    ("leaf_dfs",  # round trip: yes (tree kinds 1-3 have leaves whose BFS and DFS ids differ)
     lambda: M.Frame(120, 40, _bfs(("split", 3, 50, ("split", 2, 20, ("leaf", 1, 0, 0, 0), ("leaf", 2, 0, 0, 0)),
                                    ("leaf", 5, 3, 0, 0)))), M.picture_chooser(7)),
    ("make_pixel_saturate",  # round trip: no (8-bit samples never wrap)
     lambda: M.Frame(120, 40, [("leaf", 1, M.I32_MAX, 0, 0)]), M.picture_chooser(8, p_small=0.3)),
    ("palette_negative_sign",  # round trip: no (the writer's palette never uses negative indices)
     lambda: M.Frame(60, 40, [("leaf", 0, 0, 0, 0)], palette=(10, M.index_chooser(14, 10))), M.picture_chooser(10)),
    ("wp_header_ignored",  # round trip: no (the writer only writes the default WeightedHeader)
     lambda: M.Frame(120, 40, [("leaf", 6, 0, 0, 0)], global_wp=(3, 5, 1, 2, 3, 4, 5, 1, 2, 3, 4)), M.picture_chooser(9)),
]


@pytest.mark.parametrize("fault,factory,chooser", FAULTS, ids=[f[0] for f in FAULTS])
def test_planted_fault_is_caught(fault, factory, chooser):
    frame = factory()
    frame.faults = (fault,)
    assert _fault_caught(frame, chooser), fault
    clean = factory()
    assert not _fault_caught(clean, M.picture_chooser(len(fault))), "the clean model must match"


# ---------------------------------------------------------------------------------------------------------------------
# What the reference's real Modular fixtures reach
# ---------------------------------------------------------------------------------------------------------------------
# From their trees and headers (oracle jxo_modular_features; Squeeze steps are counted as applied, defaults filled in).
# Next to the matrix above they show what the ANS-checksum self-verification of those files can and cannot speak for:
# predictors 1, 3, 4, 8, 10, 11, 12, 13 and properties 3, 16..19 and 21..27 appear in none of them, no WeightedHeader is
# custom, no group has a local tree or local transform, and only the RCT types 6 and 26 occur.
FIXTURE_FEATURES = {
    'green_queen_modular_e3.jxl': {"predictors": [6], "split_properties": [15], "offset_leaves": 0, "multiplier_leaves": 0, "global_transforms": ["rct6"], "local_transforms": 0, "custom_wp_headers": 0, "local_trees": 0, "prefix": False, "lz77": False, "group_dim": 256, "groups": 6, "grey": False, "orientation": 1},
    'lz77_flower.jxl': {"predictors": [5, 6], "split_properties": [0, 2, 9, 10, 11, 12, 13, 14, 15], "offset_leaves": 0, "multiplier_leaves": 0, "global_transforms": [], "local_transforms": 0, "custom_wp_headers": 0, "local_trees": 0, "prefix": False, "lz77": True, "group_dim": 1024, "groups": 1, "grey": False, "orientation": 1},
    'delta_palette.jxl': {"predictors": [5, 6], "split_properties": [1, 9, 10, 11, 12, 13, 15], "offset_leaves": 0, "multiplier_leaves": 0, "global_transforms": ["palette(c=3,colors=0,deltas=0,pred=13)"], "local_transforms": 0, "custom_wp_headers": 0, "local_trees": 0, "prefix": False, "lz77": False, "group_dim": 256, "groups": 9, "grey": False, "orientation": 1},
    'grayscale_public_university.jxl': {"predictors": [0], "split_properties": [0, 1, 4, 5, 6, 7, 8, 15], "offset_leaves": 0, "multiplier_leaves": 90, "global_transforms": ["squeeze(17 steps)"], "local_transforms": 0, "custom_wp_headers": 0, "local_trees": 0, "prefix": False, "lz77": False, "group_dim": 256, "groups": 84, "grey": True, "orientation": 1},
    'tree_max_property_20.jxl': {"predictors": [2, 7, 9], "split_properties": [9, 20], "offset_leaves": 3, "multiplier_leaves": 0, "global_transforms": ["rct6"], "local_transforms": 0, "custom_wp_headers": 0, "local_trees": 0, "prefix": True, "lz77": False, "group_dim": 1024, "groups": 1, "grey": False, "orientation": 7},
    'issue865_large_toc.jxl': {"predictors": [5], "split_properties": [], "offset_leaves": 0, "multiplier_leaves": 0, "global_transforms": ["rct6"], "local_transforms": 0, "custom_wp_headers": 0, "local_trees": 0, "prefix": True, "lz77": False, "group_dim": 128, "groups": 1806, "grey": False, "orientation": 1},
    '3x3_srgb_lossless.jxl': {"predictors": [6], "split_properties": [], "offset_leaves": 0, "multiplier_leaves": 0, "global_transforms": ["rct26"], "local_transforms": 0, "custom_wp_headers": 0, "local_trees": 0, "prefix": True, "lz77": False, "group_dim": 512, "groups": 1, "grey": False, "orientation": 1},
}


def modular_features(data):
    import ctypes as C
    import json
    from tests import oracle_binding as ob
    lib = ob._load_modular()
    lib.jxo_modular_features.restype = C.c_int64
    lib.jxo_modular_features.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
    buf = C.create_string_buffer(1 << 16)
    n = lib.jxo_modular_features(data, len(data), buf, len(buf))
    if n < 0:
        raise abi.JxgError(int(n), lib.jxo_modular_last_error().decode())
    return json.loads(buf.value.decode())


@pytest.mark.parametrize("name", sorted(FIXTURE_FEATURES))
def test_real_fixture_features(golden_dir, name):
    import os
    data = open(os.path.join(golden_dir, "jxl", name), "rb").read()
    assert modular_features(data) == FIXTURE_FEATURES[name]


def test_token_frames_reach_what_the_fixtures_do_not():
    """The token-level matrix uses, between its frames, every predictor and split property 0..27 that the fixtures
    leave out, custom WeightedHeaders, local trees and local transforms (read back from the written files)."""
    feats = [modular_features(model(n)[1]) for n in CASES]
    assert set().union(*(f["predictors"] for f in feats)) == set(range(14))
    assert set().union(*(f["split_properties"] for f in feats)) >= set(range(28))
    assert sum(f["custom_wp_headers"] for f in feats) > 0 and sum(f["local_trees"] for f in feats) > 0
    assert sum(f["local_transforms"] for f in feats) >= 42
