"""Region decode of Modular frames on the GPU (jxg_modular_batch_add_region): every region equals, byte for byte, the
crop of the whole-frame GPU decode and of the CPU oracle, for host and device outputs, padded strides, 1, 2 and 4
lanes per warp and every orientation; only the group streams of the cone are decoded (other sections can hold
anything, and the walk and LZ77 statistics count exactly the selected streams); a failing stream inside the cone is
reported by its whole-frame group; mixed batches, SM budgets and poisoned context pools give the same bytes."""
import os

import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import modular_ref as M
from tests import test_modular_lz77 as L
from tests import test_modular_ref as T
from tests import test_modular_squeeze as S
from tests import test_modular_walk_table as WT

pytestmark = pytest.mark.gpu

FIXTURES = ["green_queen_modular_e3.jxl", "grayscale_public_university.jxl", "issue865_large_toc.jxl",
            "3x3_srgb_lossless.jxl", "lz77_flower.jxl", "tree_max_property_20.jxl"]
_ORACLE = {}


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


def _fixture(golden_dir, name):
    return open(os.path.join(golden_dir, "jxl", name), "rb").read()


def _oracle(data):
    key = hash(data)
    if key not in _ORACLE:
        from tests import oracle_binding as ob
        _ORACLE[key] = ob.decode_modular_file(data)
    return _ORACLE[key]


def _regions(w, h, seed, n=4):
    rng = np.random.default_rng(seed)
    out = [(0, 0, 1, 1), (w - 1, h - 1, 1, 1), (w - 1, 0, 1, 1), (0, h - 1, 1, 1), (0, 0, w, h), (0, h // 2, w, 1),
           (w // 2, 0, 1, h)]
    for _ in range(n):
        x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
        out.append((x, y, int(rng.integers(1, min(w - x, 300) + 1)), int(rng.integers(1, min(h - y, 300) + 1))))
    return out


def decode(ctx, items, lanes=1, device=False, pad=0, stats=False, expect_error=False):
    """items: [(ModularParsedFrame, region or None)] as one batch. Returns the outputs (h x w x 3 u8), then the
    batch's walk_stats() and lz77_stats() when asked for, then (frame, group) of a failing stream when expected."""
    import torch
    import jxl_rs_b200 as j
    b = j.ModularBatch(ctx, lanes)
    bufs = []
    try:
        for fr, reg in items:
            w, h = (fr.width, fr.height) if reg is None else (reg[2], reg[3])
            stride = w * 3 + pad
            if device:
                t = torch.full((h * stride,), 0xA5, dtype=torch.uint8, device=f"cuda:{ctx.device}")
            else:
                t = torch.full((h * stride,), 0xA5, dtype=torch.uint8).pin_memory()
            bufs.append((t, w, h, stride))
            b.add(fr, t.data_ptr(), stride, device, region=reg)
        st = (b.walk_stats(), b.lz77_stats())
        b.run()
        bad = None
        if expect_error:
            import ctypes as C
            bf, bg = C.c_uint32(), C.c_uint32()
            r = b._lib.jxg_modular_batch_wait(b._h, C.byref(bf), C.byref(bg))
            bad = (r, bf.value, bg.value)
        else:
            b.wait()
        outs = []
        for t, w, h, stride in bufs:
            a = t.cpu().numpy().reshape(h, stride)
            if pad:
                assert (a[:, w * 3:] == 0xA5).all(), "bytes past the row were written"
            outs.append(np.ascontiguousarray(a[:, :w * 3]).reshape(h, w, 3))
    finally:
        b.close()
    res = (outs,)
    if stats:
        res += st
    if expect_error:
        res += (bad,)
    return res


def _crop(img, r):
    return img[r[1]:r[1] + r[3], r[0]:r[0] + r[2]]


def check_regions(ctx, data, seed, lanes=1, device=False, pad=0, n=4):
    import jxl_rs_b200 as j
    fr = j.ModularParsedFrame(data)
    regs = _regions(fr.width, fr.height, seed, n)
    (outs,) = decode(ctx, [(fr, None)] + [(fr, r) for r in regs], lanes, device, pad)
    whole, ref = outs[0], _oracle(data)
    assert np.array_equal(whole, ref)
    for r, o in zip(regs, outs[1:]):
        assert np.array_equal(o, _crop(whole, r)), r
        assert np.array_equal(o, _crop(ref, r)), r


# (lanes, device output, row padding) rotated over the frames so that each frame meets one and the set meets all
MODES = [(1, False, 0), (2, True, 0), (4, False, 5), (1, True, 7), (2, False, 1), (4, True, 3)]


@pytest.mark.parametrize("k,name", list(enumerate(FIXTURES)))
def test_fixtures(ctx, golden_dir, k, name):
    lanes, device, pad = MODES[k % len(MODES)]
    check_regions(ctx, _fixture(golden_dir, name), k, lanes, device, pad)


def _token_sets():
    out = [("ref", n, lambda n=n: T.model(n)[1]) for n in T.CASES]
    out += [("squeeze", n, lambda n=n: S.model(n)[1]) for n in S.CASES if n != "local_squeeze"]
    out += [("lz77", n, lambda n=n: L.token_frame(n, 2)[1]) for n in L.TOKEN_CASES]
    out += [("walk", n, lambda n=n: [d for _, d in WT.items(n)]) for n in WT.CASES]
    return out


TOKEN_SETS = _token_sets()


@pytest.mark.parametrize("k", range(len(TOKEN_SETS)), ids=[f"{s}-{n}" for s, n, _ in TOKEN_SETS])
def test_token_frames(ctx, k):
    kind, name, get = TOKEN_SETS[k]
    data = get()
    lanes, device, pad = MODES[k % len(MODES)]
    for i, d in enumerate(data if isinstance(data, list) else [data]):
        check_regions(ctx, d, k * 10 + i, lanes, device, pad, n=3)


@pytest.mark.parametrize("orientation", range(1, 9))
def test_orientations(ctx, orientation):
    """Writer frames (RCT + Squeeze, groups of 128) in every orientation."""
    rng = np.random.default_rng(orientation)
    f = M.Frame(300, 170, M.random_tree(rng, 4, [0, 1, 3, 6, 9]), group_shift=0, orientation=orientation,
                transforms=[("rct", 0, 6), ("squeeze", [])])
    f.decode(M.picture_chooser(orientation, p_small=0.2))
    import synth
    data = synth.encode_modular_tokens(f.spec)
    check_regions(ctx, data, orientation, *MODES[orientation % len(MODES)], n=6)


# ---------------------------------------------------------------------------------------------------------------------
# Only the cone is decoded
# ---------------------------------------------------------------------------------------------------------------------
def _frame_with_other_sections(frame, keep_groups, seed):
    """The written frame with the tokens of every HF section outside `keep_groups` replaced by seeded random values."""
    import synth
    rng = np.random.default_rng(seed)
    spec = dict(frame.spec)
    secs = list(spec["sections"])
    n_hf = len(M.channel_sections([{"w": frame.w, "h": frame.h, "shift": (0, 0)}], frame.w, frame.h,
                                  frame.group_shift)[2])
    first_hf = len(secs) - n_hf
    for g in range(n_hf):
        s = secs[first_hf + g]
        if g in keep_groups or s is None or s.get("tokens") is None:
            continue
        s = dict(s)
        s["tokens"] = [(c, int(rng.integers(0, 1 << 12))) for c, _ in s["tokens"]]
        secs[first_hf + g] = s
    spec["sections"] = secs
    return synth.encode_modular_tokens(spec)


def test_sections_outside_the_cone_are_not_read(ctx):
    import jxl_rs_b200 as j
    for name, (frame, data) in [("squeeze", S.model("default_rgb_groups")), ("rct", T.model("edge_rects_128")),
                                ("palette", T.model("palette_groups"))]:
        fr = j.ModularParsedFrame(data)
        for k, reg in enumerate(_regions(fr.width, fr.height, len(name), 3)):
            groups, _, _ = fr.region_plan(reg)
            other = j.ModularParsedFrame(_frame_with_other_sections(frame, set(groups), k))
            (a, b) = decode(ctx, [(fr, reg), (other, reg)])[0]
            assert np.array_equal(a, b), (name, reg)


def test_stats_count_the_selected_streams(ctx, golden_dir):
    """walk_stats counts the non-empty rects of the selected streams and nothing else (every rect of the token frame
    below takes the single-leaf walk); lz77_stats counts the selected LZ77 streams."""
    import jxl_rs_b200 as j
    frame = M.Frame(300, 270, [("leaf", 5, 0, 0, 0)], group_shift=0)
    frame.decode(M.picture_chooser(3))
    import synth
    fr = j.ModularParsedFrame(synth.encode_modular_tokens(frame.spec))
    for reg in [(0, 0, 1, 1), (120, 120, 20, 20), (0, 0, 300, 270), (299, 0, 1, 270)]:
        groups, _, _ = fr.region_plan(reg)
        _, walks, _ = decode(ctx, [(fr, reg)], stats=True)
        assert walks["single_leaf"] + walks["generic"] + sum(walks["by_property"].values()) == 3 * len(groups)
    lz_frame, lz_data, _ = L.token_frame("ans_tree", 1)
    fr = j.ModularParsedFrame(lz_data)
    for reg in [(0, 0, 1, 1), (0, 0, fr.width, fr.height), (fr.width - 1, fr.height - 1, 1, 1)]:
        groups, _, _ = fr.region_plan(reg)
        _, _, lz = decode(ctx, [(fr, reg)], stats=True)
        assert lz["lz77_streams"] == len(groups), (reg, lz, groups)


def test_failing_stream_is_named_by_its_whole_frame_group(ctx):
    """A stream that starts with an LZ77 copy fails with JXG_ERR_LZ77: inside the cone wait names (frame, group of the
    whole frame); outside it the region decodes and wait returns OK."""
    import jxl_rs_b200 as j
    frame = L.token_frame("ans_tree", 1)[0]
    n_lf = 1
    for g_bad in (0, 5):
        _, data, _ = L.token_frame("ans_tree", 1, fault=(1, 1 + n_lf + g_bad))
        fr = j.ModularParsedFrame(data)
        good = j.ModularParsedFrame(L.token_frame("ans_tree", 1)[1])
        in5 = (260, 130, 5, 5)  # group 5 of the 3 x 3 grid of 128 x 128 groups
        reg_in = in5 if g_bad == 5 else (0, 0, 5, 5)
        reg_out = (0, 0, 5, 5) if g_bad == 5 else in5
        assert g_bad in fr.region_plan(reg_in)[0] and g_bad not in fr.region_plan(reg_out)[0]
        outs, bad = decode(ctx, [(good, None), (fr, reg_out), (fr, reg_in)], expect_error=True)
        assert bad == (-10, 2, g_bad), bad
        outs = decode(ctx, [(good, None), (fr, reg_out)])[0]
        assert np.array_equal(outs[1], _crop(outs[0], reg_out))


# ---------------------------------------------------------------------------------------------------------------------
# Mixed batches, SM budgets, stale memory, taps and the Python entry points
# ---------------------------------------------------------------------------------------------------------------------
def _mixed(ctx, golden_dir, lanes=2):
    import jxl_rs_b200 as j
    q = j.ModularParsedFrame(_fixture(golden_dir, "green_queen_modular_e3.jxl"))
    # Squeeze, then RCT in header order: the inverse plan starts with the RCT, so the RCT-only frames' step lists are
    # prefixes of its own
    sq = j.ModularParsedFrame(S.model("squeeze_then_rct")[1])
    rct = j.ModularParsedFrame(T.model("groups_256")[1])
    W, H = q.width, q.height
    items = [(q, None), (q, (W // 8, H // 8, W // 2, H // 2)), (q, (W // 4, H // 4, W // 2, H // 2)), (sq, (10, 3, 40, 30)),
             (rct, None), (sq, None), (rct, (260, 290, 10, 10)), (q, (0, 0, W, H))]
    return items, decode(ctx, items, lanes)[0]


def test_mixed_batches(ctx, golden_dir):
    import jxl_rs_b200 as j
    items, outs = _mixed(ctx, golden_dir)
    for (fr, reg), o in zip(items, outs):
        alone = decode(ctx, [(fr, None)])[0][0]
        assert np.array_equal(o, alone if reg is None else _crop(alone, reg)), reg
    ctx.set_sm_budget(1)
    try:
        _, outs1 = _mixed(ctx, golden_dir, lanes=4)
    finally:
        ctx.set_sm_budget(0)
    for a, b in zip(outs, outs1):
        assert np.array_equal(a, b)
    # a refused region leaves the batch as it was
    b = j.ModularBatch(ctx)
    try:
        import torch
        t = torch.empty(100, dtype=torch.uint8).pin_memory()
        q = items[0][0]
        with pytest.raises(abi.JxgError) as e:
            b.add(q, t.data_ptr(), 30, False, region=(0, 0, 0, 1))
        assert e.value.code == -22
        with pytest.raises(abi.JxgError) as e:
            b.add(q, t.data_ptr(), 29, False, region=(0, 0, 10, 1))
        assert e.value.code == -9
        assert b.walk_stats()["generic"] + b.walk_stats()["single_leaf"] == 0
        b.add(q, t.data_ptr(), 30, False, region=(0, 0, 10, 1))
    finally:
        b.close()


@pytest.mark.parametrize("fill", [0xFF, 0x7F])
def test_poisoned_pools(ctx, golden_dir, fill):
    import jxl_rs_b200 as j
    items, fresh = _mixed(ctx, golden_dir)
    sq = j.ModularParsedFrame(_fixture(golden_dir, "grayscale_public_university.jxl"))
    regs = [(sq, r) for r in _regions(sq.width, sq.height, 3, 3)]
    fresh_sq = decode(ctx, regs)[0]
    ctx.set_pool_fill(fill)
    try:
        _, poisoned = _mixed(ctx, golden_dir)
        poisoned_sq = decode(ctx, regs)[0]
    finally:
        ctx.set_pool_fill(-1)
    for a, b in zip(fresh + fresh_sq, poisoned + poisoned_sq):
        assert np.array_equal(a, b)


def test_read_planes_refuses_a_region_frame(ctx, golden_dir):
    import torch
    import jxl_rs_b200 as j
    fr = j.ModularParsedFrame(_fixture(golden_dir, "3x3_srgb_lossless.jxl"))
    b = j.ModularBatch(ctx)
    try:
        t = torch.empty(64, dtype=torch.uint8).pin_memory()
        b.add(fr, t.data_ptr(), 9, False)
        b.add(fr, t.data_ptr() + 32, 6, False, region=(1, 1, 2, 2))
        b.run()
        b.wait()
        assert b.read_planes(0).shape == (3, 3, 3)
        with pytest.raises(abi.JxgError) as e:
            b.read_planes(1)
        assert e.value.code == -22
    finally:
        b.close()


def test_python_entry_points(ctx, golden_dir):
    import torch
    import jxl_rs_b200 as j
    data = _fixture(golden_dir, "lz77_flower.jxl")
    fr = j.ModularParsedFrame(data)
    groups, arena, need = fr.region_plan((5, 6, 40, 30))
    assert groups == [] and len(arena) == len(need)  # one group: every channel is small, decoded in section 0
    out = torch.empty((30, 40, 3), dtype=torch.uint8, device="cuda:0")
    b = j.ModularBatch(ctx)
    try:
        b.add(fr, out.data_ptr(), 40 * 3, True, region=(5, 6, 40, 30))
        b.run()
        b.wait()
    finally:
        b.close()
    assert np.array_equal(out.cpu().numpy(), _crop(_oracle(data), (5, 6, 40, 30)))
