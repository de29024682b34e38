"""Region decode of Modular frames without a GPU: the dependency cone the library plans for a region
(ModularParsedFrame.region_plan, jxg_modular_parsed_region_plan) against a Python restatement built on the channel ->
section rules of tests/modular_ref.py, and the refusals of jxg_modular_batch_add_region, each with a valid twin.

The restatement walks the global transforms in header order (meta-apply order), which is the inverse plan backwards:
each channel of the list carries the rectangle the region needs of it, from the output channels (the coded rectangle
of the region) to the coded channels, whose rects in the HF group grid select the group streams. It shares no code
with the C++ (csrc/host/modular_region.cc); its unsqueeze rule is derived from the set of outputs a pair loop from
column 0 must produce."""
import os

import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import modular_ref as M
from tests import test_modular_lz77 as L
from tests import test_modular_ref as T
from tests import test_modular_squeeze as S
from tests import test_modular_walk_table as WT
from tests.f64_pipeline import orient

EMPTY = (0, 0, 0, 0)


# ---------------------------------------------------------------------------------------------------------------------
# The restatement
# ---------------------------------------------------------------------------------------------------------------------
def _union(a, b):
    if a == EMPTY:
        return b
    if b == EMPTY:
        return a
    return (min(a[0], b[0]), min(a[1], b[1]), max(a[2], b[2]), max(a[3], b[3]))


def _rect(x0, y0, x1, y1):
    return (x0, y0, x1, y1) if x0 < x1 and y0 < y1 else EMPTY


class _Buf:
    """One plan buffer: a channel of the list at some stage of meta-apply, with the rectangle the region needs of it."""

    def __init__(self, w, h, shift):
        self.w, self.h, self.shift, self.need, self.id = w, h, shift, EMPTY, None


def _unsqueeze_needs(out, n_out, n_avg, n_res):
    """Along the squeezed axis: an output range [0, end) (end = out's far edge) is made by the pair loop from index 0.
    Pair k writes outputs 2k and 2k + 1 from avg[k], res[k] and the next average avg[min(k + 1, n_avg - 1)]; an odd
    output length ends with the tail output avg[n_avg - 1]. Returns (avg indices read, residual indices read) as
    half-open ends, from the outputs the range holds."""
    end = out
    pairs = sum(1 for k in range(n_res) if 2 * k < end)
    avg_read = {0} if n_avg else set()
    if pairs:
        avg_read |= {pairs - 1, min(pairs, n_avg - 1)}
    if (n_avg + n_res) % 2 and end == n_out:
        avg_read.add(n_avg - 1)
    return (max(avg_read) + 1 if avg_read else 0), pairs


def restated_cone(w, h, grey, group_shift, transforms, coded):
    """(groups, {buffer id: need}) of the coded rectangle `coded` of a frame: w x h coded, `transforms` in header order
    as modular_ref.Frame takes them (Squeeze steps [] for the default list)."""
    nc = 1 if grey else 3
    chans = [_Buf(w, h, (0, 0)) for _ in range(nc)]
    for b in chans:
        b.need = coded
    made = []  # per transform, the buffers its inverse writes, in the inverse plan's order
    for t in transforms:
        if t[0] == "rct":
            b = t[1]
            u = EMPTY
            for c in chans[b:b + 3]:
                u = _union(u, c.need)
            for c in chans[b:b + 3]:
                c.need = u
            made.append([])
        elif t[0] == "palette":
            _, b, n, ncol = t
            outs = chans[b:b + n]
            index = _Buf(outs[0].w, outs[0].h, outs[0].shift)
            for o in outs:
                index.need = _union(index.need, o.need)
            pal = _Buf(ncol, n, None)
            pal.need = _rect(0, 0, ncol, n)
            chans = [pal] + chans[:b] + [index] + chans[b + n:]
            made.append([outs])
        else:
            shapes = [{"w": c.w, "h": c.h, "shift": c.shift} for c in chans]
            steps = M.meta_apply_squeeze(shapes, list(t[1]), M.Coverage())
            per_step = []
            for hz, in_place, b, n in steps:
                off = b + n if in_place else len(chans)
                outs = chans[b:b + n]
                res = []
                for ic, o in enumerate(outs):
                    sh = None if o.shift is None else ((o.shift[0] + 1, o.shift[1]) if hz else (o.shift[0], o.shift[1] + 1))
                    if hz:
                        aw = -(-o.w // 2)
                        avg, r = _Buf(aw, o.h, sh), _Buf(o.w - aw, o.h, sh)
                    else:
                        ah = -(-o.h // 2)
                        avg, r = _Buf(o.w, ah, sh), _Buf(o.w, o.h - ah, sh)
                    if o.need != EMPTY:
                        x0, y0, x1, y1 = o.need
                        if hz:
                            ae, re_ = _unsqueeze_needs(x1, o.w, avg.w, r.w)
                            avg.need, r.need = _rect(0, y0, ae, y1), _rect(0, y0, re_, y1)
                        else:
                            ae, re_ = _unsqueeze_needs(y1, o.h, avg.h, r.h)
                            avg.need, r.need = _rect(x0, 0, x1, ae), _rect(x0, 0, x1, re_)
                    chans[b + ic] = avg
                    res.append(r)
                chans[off:off] = res
                per_step.append(outs)
            made.append(per_step[::-1])
    for i, c in enumerate(chans):
        c.id = i
    nxt = len(chans)
    for group in reversed(made):
        for outs in group:
            for o in outs:
                o.id, nxt = nxt, nxt + 1
    needs = {c.id: c.need for c in chans}
    for group in made:
        for outs in group:
            needs.update({o.id: o.need for o in outs})
    shapes = [{"w": c.w, "h": c.h, "shift": c.shift} for c in chans]
    _, _, hf = M.channel_sections(shapes, w, h, group_shift)
    groups, rects = [], {}
    for g, (_, items) in enumerate(hf):
        hit = False
        for i, (x0, y0, rw, rh) in items:
            n = needs[i]
            if rw and rh and n != EMPTY and x0 < n[2] and n[0] < x0 + rw and y0 < n[3] and n[1] < y0 + rh:
                hit = True
        if hit:
            groups.append(g)
            rects[g] = [(i, (x0, y0, x0 + rw, y0 + rh)) for i, (x0, y0, rw, rh) in items if rw and rh]
    return groups, needs, rects


# ---------------------------------------------------------------------------------------------------------------------
# Frames and regions
# ---------------------------------------------------------------------------------------------------------------------
class Geo:
    """What the restatement needs of a frame: coded size, grey, group shift, orientation, header-order transforms."""

    def __init__(self, w, h, grey, group_shift, orientation, transforms):
        self.w, self.h, self.grey, self.group_shift, self.o, self.transforms = w, h, grey, group_shift, orientation, transforms
        self._disp = None

    @property
    def disp_size(self):
        return (self.h, self.w) if self.o >= 5 else (self.w, self.h)

    def coded_rect(self, region):
        """The coded rectangle of a display region: the coded pixels the oriented image shows there."""
        if self._disp is None:
            self._disp = orient(np.arange(self.w * self.h, dtype=np.int64).reshape(self.h, self.w), self.o)
        x, y, rw, rh = region
        v = self._disp[y:y + rh, x:x + rw]
        lo, hi = int(v.min()), int(v.max())
        xs, ys = (lo % self.w, hi % self.w), (lo // self.w, hi // self.w)
        # the corners of a rectangle: min and max of the flat index are opposite corners
        return (min(xs), min(ys), max(xs) + 1, max(ys) + 1)

    def display_region(self, coded):
        """The display region showing coded rectangle `coded` (x0, y0, x1, y1)."""
        m = np.zeros((self.h, self.w), bool)
        m[coded[1]:coded[3], coded[0]:coded[2]] = True
        d = orient(m, self.o)
        ys, xs = np.nonzero(d)
        return (int(xs.min()), int(ys.min()), int(xs.max() - xs.min() + 1), int(ys.max() - ys.min() + 1))


def model_geo(frame):
    nc = 1 if frame.grey else 3
    return Geo(frame.w, frame.h, frame.grey, frame.group_shift, frame.orientation, frame._global_transforms(nc))


def fixture_geo(data):
    from tests import oracle_binding as ob
    f = T.modular_features(data)
    dw, dh, _, _ = ob.modular_info(data)
    w, h = (dh, dw) if f["orientation"] >= 5 else (dw, dh)
    tr = []
    for t in f["global_transforms"]:
        if t.startswith("rct"):
            tr.append(("rct", 0, int(t[3:])))
        elif t.startswith("squeeze"):
            tr.append(("squeeze", []))
        else:
            raise AssertionError(t)
    return Geo(w, h, f["grey"], int(np.log2(f["group_dim"] // 128)), f["orientation"], tr)


def regions(geo, seed, n_random=4):
    """Display regions: the full frame, 1 x 1 at each corner, a row, a column, seeded random ones, rectangles
    straddling group edges, and rectangles ending on both sides of every power of two (the pair boundaries of every
    Squeeze level), the last two given in coded coordinates."""
    W, H = geo.disp_size
    rng = np.random.default_rng(seed)
    out = {(0, 0, W, H), (0, 0, 1, 1), (W - 1, 0, 1, 1), (0, H - 1, 1, 1), (W - 1, H - 1, 1, 1),
           (0, H // 2, W, 1), (W // 2, 0, 1, H)}
    for _ in range(n_random):
        x, y = int(rng.integers(0, W)), int(rng.integers(0, H))
        out.add((x, y, int(rng.integers(1, W - x + 1)), int(rng.integers(1, H - y + 1))))
    gd = 128 << geo.group_shift
    coded = []
    for k in range(1, 3):
        if k * gd < geo.w:
            coded.append((k * gd - 3, 0, min(geo.w, k * gd + 2), min(geo.h, 5)))
        if k * gd < geo.h:
            coded.append((max(0, geo.w - 7), k * gd - 1, geo.w, min(geo.h, k * gd + 1)))
    p = 2
    while p <= max(geo.w, geo.h):
        for e in (p - 1, p, p + 1):
            x1, y1 = min(max(e, 1), geo.w), min(max(e, 1), geo.h)
            coded.append((max(0, x1 - 2), max(0, y1 - 3), x1, y1))
        p *= 2
    for c in coded:
        out.add(geo.display_region(c))
    return sorted(out)


def check_plan(parsed, geo, region):
    groups, arena, need = parsed.region_plan(region)
    r_groups, r_need, r_rects = restated_cone(geo.w, geo.h, geo.grey, geo.group_shift, geo.transforms,
                                              geo.coded_rect(region))
    assert groups == r_groups, (region, groups, r_groups)
    assert len(need) == len(r_need), (region, len(need), len(r_need))
    for i, n in enumerate(need):
        assert n == r_need[i], (region, i, n, r_need[i])
        if n != EMPTY:
            assert _union(arena[i], n) == arena[i], (region, i)
    for g in groups:
        for i, r in r_rects[g]:
            assert _union(arena[i], r) == arena[i], (region, g, i, r, arena[i])
    return groups


def _parsed(data):
    import jxl_rs_b200 as j
    return j.ModularParsedFrame(data)


def _device_frame(data):
    """The parsed frame, or None when jxg_modular_batch_add refuses the frame (then every region is refused alike)."""
    p = _parsed(data)
    try:
        p.region_plan((0, 0, p.width, p.height))
    except abi.JxgError as e:
        assert e.code == -2, e
        with pytest.raises(abi.JxgError) as e2:
            p.region_plan((0, 0, 1, 1))
        assert e2.value.code == -2
        return None
    return p


def _check_model(frame, data, seed):
    p = _device_frame(data)
    if p is None:
        return 0
    geo = model_geo(frame)
    for r in regions(geo, seed):
        check_plan(p, geo, r)
    return 1


# ---------------------------------------------------------------------------------------------------------------------
# Token-level frames
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", T.CASES)
def test_plan_token_frames(name):
    frame, data = T.model(name)
    assert _check_model(frame, data, len(name))


@pytest.mark.parametrize("name", S.CASES)
def test_plan_squeeze_frames(name):
    frame, data = S.model(name)
    checked = _check_model(frame, data, len(name) + 1)
    assert checked == (name != "local_squeeze")  # a group-local Squeeze is refused


@pytest.mark.parametrize("name", L.TOKEN_CASES)
def test_plan_lz77_frames(name):
    frame, data, _ = L.token_frame(name, 1)
    assert _check_model(frame, data, len(name) + 2)


@pytest.mark.parametrize("name", WT.CASES)
def test_plan_walk_table_frames(name):
    for it, data in WT.items(name):
        assert _check_model(it.frame, data, len(name) + 3)


FIXTURES = ["green_queen_modular_e3.jxl", "grayscale_public_university.jxl", "issue865_large_toc.jxl",
            "3x3_srgb_lossless.jxl", "lz77_flower.jxl", "tree_max_property_20.jxl"]


@pytest.mark.parametrize("name", FIXTURES)
def test_plan_real_fixtures(golden_dir, name):
    data = open(os.path.join(golden_dir, "jxl", name), "rb").read()
    geo = fixture_geo(data)
    p = _parsed(data)
    if geo.transforms and geo.transforms[0][0] == "squeeze":  # the default list the fixture applies is the one restated
        shapes = [{"w": geo.w, "h": geo.h, "shift": (0, 0)}] * (1 if geo.grey else 3)
        n = len(M.meta_apply_squeeze([dict(s) for s in shapes], [], M.Coverage()))
        assert T.modular_features(data)["global_transforms"] == [f"squeeze({n} steps)"]
    for r in regions(geo, len(name), n_random=3 if geo.w * geo.h > 10 ** 7 else 6):
        check_plan(p, geo, r)


def test_squeeze_cone_reaches_the_top_left(golden_dir):
    """On the Squeeze fixture a bottom-right crop needs far more group streams than a top-left one of the same size:
    every unsqueeze output depends on the outputs to its left and above."""
    data = open(os.path.join(golden_dir, "jxl", "grayscale_public_university.jxl"), "rb").read()
    p = _parsed(data)
    tl, _, _ = p.region_plan((0, 0, 256, 256))
    br, _, _ = p.region_plan((p.width - 256, p.height - 256, 256, 256))
    assert len(br) > 4 * len(tl), (len(tl), len(br))
    assert p.info.num_groups == 84


# ---------------------------------------------------------------------------------------------------------------------
# Refusals, each with its valid twin
# ---------------------------------------------------------------------------------------------------------------------
def _code(p, region):
    try:
        p.region_plan(region)
        return 0
    except abi.JxgError as e:
        return e.code


def test_region_argument_refusals():
    frame, data = T.model("groups_256")
    p = _parsed(data)
    W, H = p.width, p.height
    bad_good = [
        ((0, 0, 0, 5), (0, 0, 1, 5)),              # empty: no columns
        ((3, 3, 4, 0), (3, 3, 4, 1)),              # empty: no rows
        ((W, 0, 1, 1), (W - 1, 0, 1, 1)),          # starts right of the image
        ((0, H, 1, 1), (0, H - 1, 1, 1)),          # starts below it
        ((1, 0, W, 1), (0, 0, W, 1)),              # ends past the right edge
        ((0, 1, 1, H), (0, 0, 1, H)),              # ends past the bottom edge
        ((2, 2, 2 ** 32 - 1, 1), (2, 2, W - 2, 1)),  # wraps around u32
    ]
    for bad, good in bad_good:
        assert _code(p, bad) == -22, bad
        assert _code(p, good) == 0, good


def test_refused_frame_kinds(golden_dir):
    """Delta palettes and group-local Squeeze are refused for every region as for the whole frame, with
    JXG_ERR_UNSUPPORTED, even where the region's cone holds no stream of the refused kind. (A single-section frame
    always has its one group stream empty: every channel of a frame of one group is small, so it is in section 0.)"""
    delta = _parsed(open(os.path.join(golden_dir, "jxl", "delta_palette.jxl"), "rb").read())
    assert _code(delta, (0, 0, 1, 1)) == -2 and _code(delta, (0, 0, delta.width, delta.height)) == -2
    palette = _parsed(T.model("palette_groups")[1])  # the twin: a palette without delta entries
    assert _code(palette, (0, 0, 1, 1)) == 0
    local = _parsed(S.model("local_squeeze")[1])  # group 1 squeezes locally; group 0 does not
    assert _code(local, (0, 0, 1, 1)) == -2
    twin = _parsed(S.model("default_rgb_groups")[1])
    assert _code(twin, (0, 0, 1, 1)) == 0


def test_plan_arrays_too_small():
    import ctypes as C
    frame, data = T.model("groups_256")
    p = _parsed(data)
    lib = p._lib
    ng, nb = C.c_uint32(), C.c_uint32()
    reg = abi.JxgRegion(0, 0, p.width, p.height)
    g = (C.c_uint32 * 1)()
    assert lib.jxg_modular_parsed_region_plan(p._h, C.byref(reg), g, 1, C.byref(ng), None, 0, C.byref(nb)) == -22
    assert ng.value == 4 and nb.value == 3
    g = (C.c_uint32 * 4)()
    assert lib.jxg_modular_parsed_region_plan(p._h, C.byref(reg), g, 4, C.byref(ng), None, 0, C.byref(nb)) == 0
    assert list(g) == [0, 1, 2, 3]
