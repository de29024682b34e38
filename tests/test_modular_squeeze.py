"""Squeeze against tests/modular_ref.py, an integer restatement of squeeze.rs, meta_apply.rs and the channel -> section
rules of mod.rs, on token-level frames (synth.encode_modular_tokens): default and explicit steps, in_place true and
false, squeezes of channel sub-ranges and of the meta palette channel, Squeeze with RCT and palette in either order,
channels with shift >= 3 in ModularLF streams, 1 x N frames, residuals over the full i32 range and a group-local
Squeeze. The oracle (csrc/host/modular.cc) must return the model's planes and u8 image bit for bit. Also the Squeeze
refusals with their valid twins, planted model faults, and where the reference's i32 lane form and i64 scalar form of
unsqueeze agree. No GPU."""
import itertools

import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import modular_ref as M
from tests import test_modular_ref as T

PROPS = [0, 1, 2, 3, 6, 7, 9, 10]
# explicit steps of the sub-range case: previews of channels 1-2 not in place, all three in place, channel 2 alone,
# channels 0-1 not in place
EXPLICIT = [(True, False, 1, 2), (False, True, 0, 3), (True, True, 2, 1), (False, False, 0, 2)]


def _case(name):
    """(Frame, chooser) of one case; trees are random but fixed per case name."""
    rng = np.random.default_rng(sum(map(ord, name)))
    tree = lambda depth=4, props=PROPS, **kw: M.random_tree(rng, depth, props, **kw)  # noqa: E731
    pic = M.picture_chooser(sum(map(ord, name)) + 1, p_small=0.3)
    sq = lambda steps=(): ("squeeze", list(steps))  # noqa: E731
    if name == "default_rgb_groups":  # ragged groups of 128 with channels of shift (1,0), (1,1), (2,1)
        return M.Frame(200, 150, tree(), group_shift=0, transforms=[sq()], orientation=6), pic
    if name == "tall_grey":
        return M.Frame(40, 100, tree(), grey=True, transforms=[sq()]), pic
    if name == "two_lf_groups":  # 1030 x 40: two LF groups of 1024; the tree decides on the stream id
        t = T._bfs(("split", 1, 3, ("split", 1, 30, ("leaf", 5, 0, 0, 0), ("leaf", 2, 0, 0, 0)), ("leaf", 1, 0, 0, 0)))
        return M.Frame(1030, 40, t, group_shift=0, grey=True, transforms=[sq()]), pic
    if name == "explicit_ranges":
        return M.Frame(50, 37, tree(), transforms=[sq(EXPLICIT)], orientation=3), pic
    if name == "rct_then_squeeze":
        return M.Frame(300, 40, tree(), group_shift=0, transforms=[("rct", 0, 6), sq()]), pic
    if name == "squeeze_then_rct":
        return M.Frame(61, 45, tree(), transforms=[sq([(True, True, 0, 3), (False, False, 0, 3)]), ("rct", 0, 23)]), pic
    if name == "palette_squeeze_meta":  # palette, Squeeze of the index channel, in-place Squeeze of the palette
        return M.Frame(45, 30, tree(3, [0, 2, 6]), palette=(24, M.index_chooser(3, 24)),
                       transforms=[("palette", 0, 3, 24), sq([(True, True, 1, 1), (False, True, 1, 1)]),
                                   sq([(True, True, 0, 1)])]), pic
    if name == "one_column":  # 1 x N: a zero-width residual, then the default steps (vertical first)
        return M.Frame(1, 40, tree(), grey=True, transforms=[sq([(True, True, 0, 1)]), sq()]), pic
    if name == "one_row":  # N x 1: a zero-height residual, then the default steps
        return M.Frame(41, 1, tree(), transforms=[sq([(False, True, 0, 3)]), sq()], orientation=2), pic
    if name == "one_pixel":  # the default list is empty; explicit steps give empty residuals both ways
        return M.Frame(1, 1, tree(2), transforms=[sq(), sq([(True, True, 0, 3), (False, False, 0, 3)])]), pic
    if name == "wp_refs":  # the weighted predictor and the reference properties over squeezed channels
        t = tree(5, [15, 0, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27], leaf_preds=[6, 6, 5, 1])
        return M.Frame(60, 50, t, transforms=[sq()], global_wp=T._wp(rng)), M.picture_chooser(9, p_small=0.3)
    if name == "prefix_codes":
        return M.Frame(90, 70, tree(), prefix=True, hybrid=(2, 1, 1), transforms=[sq()]), pic
    if name == "full_range":  # residuals anywhere in the i32 range: the unsqueeze outputs wrap
        return M.Frame(40, 30, tree(), transforms=[sq()]), M.picture_chooser(5, p_small=0.1, p_huge=0.5)
    if name == "local_squeeze":  # group 1: default local Squeeze; group 3: RCT, then Squeeze not in place
        groups = {1: {"transforms": [sq()]},
                  3: {"transforms": [("rct", 0, 6), sq([(True, False, 0, 2), (False, True, 2, 1)])], "tree": tree(3)}}
        return M.Frame(200, 140, tree(), group_shift=0, groups=groups), pic
    raise KeyError(name)


CASES = ["default_rgb_groups", "tall_grey", "two_lf_groups", "explicit_ranges", "rct_then_squeeze", "squeeze_then_rct",
         "palette_squeeze_meta", "one_column", "one_row", "one_pixel", "wp_refs", "prefix_codes", "full_range",
         "local_squeeze"]
_CACHE = {}


def model(name):
    if name not in _CACHE:
        import synth
        frame, chooser = _case(name)
        frame.decode(chooser)
        _CACHE[name] = (frame, synth.encode_modular_tokens(frame.spec))
    return _CACHE[name]


def reached(cov):
    """The Squeeze features one run reached, by name."""
    r = {"tail_" + t for t in cov.tails} | {"empty_" + t for t in cov.empty_residuals} | set(cov.default_rules)
    r |= {kind for kind, _ in cov.sections}
    if cov.not_in_place:
        r.add("not_in_place")
    if cov.meta_squeezes:
        r.add("meta")
    if cov.squeeze_wrapped:
        r.add("wrapped")
    if any(b in ("increasing", "decreasing") and f for b, _, f in cov.tendency):
        r.add("clamped")
    return r


# What each case must reach, so that a change of seed cannot quietly empty it: Squeeze features, and for some the
# (section kind, shift) pairs of their coded channels
REACH = {
    "default_rgb_groups": ({"preview420", "alternating", "not_in_place", "hf", "global", "clamped"},
                           {("hf", (1, 0)), ("hf", (1, 1)), ("hf", (2, 1))}),
    "tall_grey": ({"vertical_first", "alternating", "tail_v"}, set()),
    "two_lf_groups": ({"alternating", "lf", "hf", "global"}, {("lf", (3, 3)), ("hf", (3, 2)), ("hf", (2, 2)), ("hf", (1, 0))}),
    "explicit_ranges": ({"not_in_place", "tail_h", "tail_v"}, set()),
    "rct_then_squeeze": ({"preview420", "hf"}, set()),
    "squeeze_then_rct": ({"not_in_place", "tail_h", "tail_v"}, set()),
    "palette_squeeze_meta": ({"meta", "tail_h"}, set()),
    "one_column": ({"empty_h", "vertical_first"}, set()),
    "one_row": ({"empty_v", "alternating", "tail_h"}, set()),
    "one_pixel": ({"empty_h", "empty_v", "not_in_place"}, set()),
    "wp_refs": ({"preview420", "clamped"}, set()),
    "prefix_codes": ({"alternating"}, set()),
    "full_range": ({"wrapped", "clamped"}, set()),
    "local_squeeze": ({"alternating", "not_in_place", "hf"}, set()),
}


@pytest.mark.parametrize("name", CASES)
def test_model_equals_oracle(name):
    frame, data = model(name)
    out, planes = T.oracle_planes(data)
    assert np.array_equal(planes.reshape(-1), T.model_planes(frame).reshape(-1).astype(np.int32))
    assert np.array_equal(out, frame.u8)
    feats, sections = REACH[name]
    assert feats <= reached(frame.cov), sorted(feats - reached(frame.cov))
    assert sections <= frame.cov.sections, sorted(sections - frame.cov.sections)


def test_matrix_reaches_every_feature():
    """Over all cases: both tendency branches with each clamp firing and not firing (and the flat case), tail columns
    and rows, zero-width and zero-height residuals, in_place = false, meta squeezes, every default rule, channels of
    shift 1-2 in HF groups and >= 3 in LF groups, wrapped outputs, group-local Squeeze, both tree splits on the stream
    id, the weighted predictor and reference properties over squeezed channels, ANS and prefix codes."""
    cov = M.Coverage()
    for name in CASES:
        cov.merge(model(name)[0].cov)
    assert cov.tendency >= {(b, k, f) for b in ("increasing", "decreasing") for k in (0, 1) for f in (False, True)}
    assert ("none", None, None) in cov.tendency
    assert cov.tails == {"h", "v"} and cov.empty_residuals == {"h", "v"}
    assert cov.not_in_place > 0 and cov.meta_squeezes > 0 and cov.squeeze_wrapped > 0
    assert cov.default_rules == {"preview420", "vertical_first", "alternating"}
    shifts = {k: {s for kk, s in cov.sections if kk == k} for k in ("global", "lf", "hf")}
    assert shifts["hf"] >= {(1, 0), (1, 1), (2, 1), (2, 2), (3, 2)} and shifts["lf"] and None in shifts["global"]
    assert all(min(s) >= 3 for s in shifts["lf"]) and all(min(s) <= 2 for s in shifts["hf"])
    assert (1, False) in cov.branches and (1, True) in cov.branches
    assert 6 in cov.predictors and cov.ref_slots == {0, 1}
    frames = [model(n)[0] for n in CASES]
    assert {f.prefix for f in frames} == {False, True}
    assert any(s and any(t["id"] == 2 for t in s["transforms"])
               for s in model("local_squeeze")[0].spec["sections"][1:])


# ---------------------------------------------------------------------------------------------------------------------
# Refusals
# ---------------------------------------------------------------------------------------------------------------------
def _pal(steps):
    return dict(palette=(8, M.index_chooser(2, 8)), transforms=[("palette", 0, 3, 8), ("squeeze", steps)])


REFUSALS = [
    # (name, size, frame kwargs of the refused frame, of its valid twin)
    ("range_past_end", (40, 3), dict(transforms=[("squeeze", [(True, True, 1, 3)])]),
     dict(transforms=[("squeeze", [(True, True, 1, 2)])])),
    ("mixes_meta_and_image", (40, 3), _pal([(True, True, 0, 2)]), _pal([(True, True, 0, 1)])),
    ("meta_not_in_place", (40, 3), _pal([(True, False, 0, 1)]), _pal([(True, True, 0, 1)])),
    ("32_horizontal", (40, 3), dict(grey=True, transforms=[("squeeze", [(True, True, 0, 1)] * 32)]),
     dict(grey=True, transforms=[("squeeze", [(True, True, 0, 1)] * 31)])),
    ("32_vertical", (3, 40), dict(grey=True, transforms=[("squeeze", [(False, True, 0, 1)] * 32)]),
     dict(grey=True, transforms=[("squeeze", [(False, True, 0, 1)] * 31)])),
]


def refusal_frame(size, kw, check):
    return M.Frame(*size, [("leaf", 5, 0, 0, 0)], check=check, **kw).decode(M.picture_chooser(3, p_small=0.5))


@pytest.mark.parametrize("name,size,bad,good", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_squeeze_refusals(name, size, bad, good):
    """check_squeeze_params (squeeze.rs:17-37) and TooManySqueezes (meta_apply.rs:111-113): the model refuses, the
    oracle refuses the written frame; the twin one step inside the rule decodes to the model."""
    import synth
    with pytest.raises(M.TreeRefused):
        refusal_frame(size, bad, True)
    T._assert_refused(synth.encode_modular_tokens(refusal_frame(size, bad, False).spec))
    f = refusal_frame(size, good, True)
    out, planes = T.oracle_planes(synth.encode_modular_tokens(f.spec))
    assert np.array_equal(planes.reshape(-1), T.model_planes(f).reshape(-1).astype(np.int32))
    assert np.array_equal(out, f.u8)


# ---------------------------------------------------------------------------------------------------------------------
# Planted faults
# ---------------------------------------------------------------------------------------------------------------------
def _pic(seed):
    return M.picture_chooser(seed, p_small=0.3)


FAULTS = [
    ("tendency_plus5", lambda: M.Frame(60, 40, [("leaf", 5, 0, 0, 0)], transforms=[("squeeze", [])])),
    ("diff_floor", lambda: M.Frame(60, 40, [("leaf", 5, 0, 0, 0)], transforms=[("squeeze", [])])),
    ("tail_wrong_row", lambda: M.Frame(41, 33, [("leaf", 5, 0, 0, 0)], transforms=[("squeeze", [])])),
    ("late_offset", lambda: M.Frame(16, 12, [("leaf", 5, 0, 0, 0)], transforms=[("squeeze", [(True, False, 0, 3)])])),
    ("no_vertical_first", lambda: M.Frame(20, 60, [("leaf", 5, 0, 0, 0)], grey=True, transforms=[("squeeze", [])])),
    ("preview_nc2", lambda: M.Frame(30, 20, [("leaf", 5, 0, 0, 0)], palette=(10, M.index_chooser(4, 10)),
                                    transforms=[("palette", 0, 2, 10), ("squeeze", [])])),
    ("residual_shift_kept", lambda: M.Frame(300, 40, [("leaf", 5, 0, 0, 0)], group_shift=0, grey=True,
                                            transforms=[("squeeze", [])])),
    ("lf_stream_id_plus1", lambda: _case("two_lf_groups")[0]),
    ("refs_size_only", lambda: M.Frame(20, 3, [("split", 17, 4), ("leaf", 1, 0, 0, 0), ("leaf", 2, 0, 0, 0)],
                                       palette=(20, M.index_chooser(5, 20)), transforms=[("palette", 0, 3, 20)])),
]


def _fault_caught(frame, chooser):
    """The faulty model either refuses a frame the oracle decodes, or writes one whose oracle planes differ from its."""
    import synth
    from tests import oracle_binding as ob
    try:
        frame.decode(chooser)
    except M.TreeRefused:
        return True  # the clean twin below must decode in the oracle
    data = synth.encode_modular_tokens(frame.spec)
    try:
        out, planes = ob.decode_modular_file(data, planes=True)
    except abi.JxgError:
        return True
    return not np.array_equal(planes.reshape(-1), T.model_planes(frame).reshape(-1).astype(np.int32))


@pytest.mark.parametrize("fault,factory", FAULTS, ids=[f[0] for f in FAULTS])
def test_planted_fault_is_caught(fault, factory):
    frame = factory()
    frame.faults = (fault,)
    assert _fault_caught(frame, _pic(len(fault))), fault
    assert not _fault_caught(factory(), _pic(len(fault))), "the clean model must match"


def test_clamp_order_does_not_matter():
    """Applying the two clamps of smooth_tendency_scalar in the other order changes nothing, so that planted fault is
    not a fault. Increasing branch, p = b - a >= 0, q = a - n >= 0, diff = (4p + 3q + 6) / 12: the first clamp fires
    only if 3q >= 20p + 6 (so q > p), after which the second fires only if q <= p; the second fires only if
    4p + 6 >= 21q (so q <= p), after which the first fires only if q > p. At most one clamp fires in either order, on
    the same diff. The decreasing branch is the mirror image. Exhaustive on a cube, random over the i32 range."""
    for b, a, n in itertools.product(range(-40, 41), repeat=3):
        assert M.smooth_tendency(b, a, n) == M.smooth_tendency(b, a, n, faults=("clamps_swapped",)), (b, a, n)
    rng = np.random.default_rng(7)
    for _ in range(20000):
        v = sorted(int(x) for x in rng.integers(M.I32_MIN, M.I32_MAX, 3, endpoint=True))
        for b, a, n in (v, v[::-1]):
            assert M.smooth_tendency(b, a, n) == M.smooth_tendency(b, a, n, faults=("clamps_swapped",)), (b, a, n)


# ---------------------------------------------------------------------------------------------------------------------
# The lane form against the scalar form
# ---------------------------------------------------------------------------------------------------------------------
LANE_BOUND = (1 << 29) - 1


def test_lane_form_equals_scalar_form_inside_the_domain():
    """unsqueeze_impl (i32 lanes, every operation wrapping) equals unsqueeze_scalar (i64, `as i32` at the end) whenever
    avg, res, next_avg and prev all lie in [-(2^29 - 1), 2^29 - 1]. Derivation, with b = avg, a = prev, c = next_avg:
      * |a - b|, |b - c|, |a - c| <= 2^30 - 2: the subtractions, their abs and the doublings 2|a - b|, 2|b - c|
        (<= 2^31 - 4) do not wrap, and for 0 <= v < 2^31, (v * 0x55555556) >> 32 == floor(v / 3);
      * x = (2 + |a - c| + floor(|a - b| / 3)) >> 2 == floor((3|a - c| + |a - b| + 6) / 12), which on a monotone
        triple is the scalar `(4a - 3c - b + 6) / 12` (its mirror with - 6 for the decreasing one); the two clamps are
        the scalar clamps on |.|, and the non-monotone triples give 0 in both. So the tendencies are equal, and
        |tendency| <= x + 1 <= (2^30 + 2^30 / 3) / 4 + 1 < 2^28.5;
      * diff = res + tendency: |diff| < 2^29 + 2^28.5 < 2^30, so diff + sign and the halving are the scalar
        `diff / 2` (truncation), |a| < 2^30 and |b| <= |a| + |diff| < 2^31: nothing wraps.
    Exhaustive on small 4-tuples, random near the domain's edges."""
    span = range(-6, 7)
    for avg, res, nxt, prev in itertools.product(span, repeat=4):
        assert M.unsqueeze_lane(avg, res, nxt, prev) == M.unsqueeze(avg, res, nxt, prev), (avg, res, nxt, prev)
    rng = np.random.default_rng(29)
    for _ in range(20000):
        v = [int(x) for x in rng.integers(-LANE_BOUND, LANE_BOUND, 4, endpoint=True)]
        for k in range(4):  # pin some inputs to the edges
            if rng.random() < 0.4:
                v[k] = int(rng.choice([-1, 1])) * (LANE_BOUND - int(rng.integers(0, 4)))
        assert M.unsqueeze_lane(*v) == M.unsqueeze(*v), v


def test_lane_form_differs_just_outside_the_domain():
    """At prev = 2^29, avg = next_avg = -2^29 the lane form doubles |prev - avg| = 2^30 into i32::MIN: its first clamp
    fires and the tendency becomes -(2^31 - 1), where the scalar form's second clamp gives 0. So ±2^29 inclusive does
    not suffice; the reference's output there depends on whether the pair falls on a SIMD lane or on the scalar tail."""
    v = (-(1 << 29), 0, -(1 << 29), 1 << 29)
    assert M.unsqueeze(*v) == (-(1 << 29), -(1 << 29))
    assert M.unsqueeze_lane(*v) != M.unsqueeze(*v)
    assert M.smooth_tendency_lane(1 << 29, -(1 << 29), -(1 << 29)) == -(1 << 31) + 1


# ---------------------------------------------------------------------------------------------------------------------
# Against the real fixtures
# ---------------------------------------------------------------------------------------------------------------------
def test_token_frames_reach_squeeze_the_fixtures_do_not():
    """The only real fixture with Squeeze (grayscale_public_university.jxl, test_modular_ref.FIXTURE_FEATURES) has one
    grey default list of 17 steps and no local transform; the token frames carry explicit and default lists of other
    lengths on RGB and grey, Squeeze with RCT and palette, and a group-local Squeeze (read back from the written files)."""
    assert "squeeze(17 steps)" in T.FIXTURE_FEATURES["grayscale_public_university.jxl"]["global_transforms"]
    feats = {n: T.modular_features(model(n)[1]) for n in CASES}
    squeezes = {t for f in feats.values() for t in f["global_transforms"] if t.startswith("squeeze")}
    assert len(squeezes) >= 6, squeezes
    assert any(len(f["global_transforms"]) >= 2 and any(t.startswith("rct") for t in f["global_transforms"])
               for f in feats.values())
    assert any(t.startswith("palette") for t in feats["palette_squeeze_meta"]["global_transforms"])
    assert feats["local_squeeze"]["local_transforms"] >= 3
    assert not any(f["grey"] for n, f in feats.items() if n == "default_rgb_groups")
