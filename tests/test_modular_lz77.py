"""LZ77 in Modular group streams (entropy_coding/decode.rs:286-330 with the distance multiplier of
modular/decode/bitstream.rs:193-202), on the CPU oracle: the synthetic writer's run-length and general copy modes
decode to the same planes as the frame without copies, token-level frames decode to the model's planes, a stream
longer than the 2^20-symbol window copies across it, and the two LZ77 errors are refused."""
import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import modular_ref as M


def flat_picture(w, h, seed=0):
    """A picture of flat regions: rectangles, a gradient band, thin text-like strokes (8-bit RGB)."""
    rng = np.random.default_rng(seed)
    img = np.full((h, w, 3), 236, np.uint8)
    for _ in range(max(4, (w * h) >> 14)):
        x0, y0 = int(rng.integers(0, w)), int(rng.integers(0, h))
        x1, y1 = min(w, x0 + int(rng.integers(8, max(9, w // 3)))), min(h, y0 + int(rng.integers(8, max(9, h // 3))))
        img[y0:y1, x0:x1] = rng.integers(0, 256, 3)
    band = slice(h // 3, h // 3 + max(1, h // 10))
    img[band, :, 0] = (np.arange(w) * 255 // max(1, w - 1)).astype(np.uint8)[None, :]
    for y in range(5, h, 23):  # strokes: one-pixel lines with gaps, like glyph rows
        img[y, (np.arange(w) % 7) < 4] = 20
    return img


def oracle(data):
    from tests import oracle_binding as ob
    return ob.decode_modular_file(data, planes=True)


@pytest.mark.parametrize("kw", [dict(rct=6, squeeze=0, tree_kind=1), dict(rct=6, squeeze=1, tree_kind=2),
                                dict(rct=0, squeeze=0, tree_kind=0), dict(rct=6, squeeze=0, tree_kind=3)],
                         ids=["rct_tree", "squeeze_wp", "gradient", "ref_props"])
@pytest.mark.parametrize("source", ["procedural", "flat"])
def test_lz77_modes_decode_to_the_same_planes(kw, source):
    import synth
    w, h = 600, 520
    src = flat_picture(w, h) if source == "flat" else None
    want = src if src is not None else synth.modular_source(w, h, 7)
    _, base = oracle(synth.encode_modular(w, h, 7, source=src, **kw))
    for lz in (1, 2):
        out, planes = oracle(synth.encode_modular(w, h, 7, source=src, lz77=lz, **kw))
        assert np.array_equal(planes, base) and np.array_equal(out, want), lz
        assert synth.lz77_census()["copies"] > 0


def test_census_reaches_every_kind_of_copy():
    import synth
    w, h = 600, 520
    c1 = None
    for squeeze in (0, 1):
        synth.encode_modular(w, h, 7, rct=6, squeeze=squeeze, source=flat_picture(w, h), lz77=1)
        c1 = synth.lz77_census()
        assert c1["copies"] > 0 and c1["plain"] == 0 and c1["max_distance"] == 1
        synth.encode_modular(w, h, 7, rct=6, squeeze=squeeze, source=flat_picture(w, h), lz77=2)
        c = synth.lz77_census()
        assert c["special"] > 0 and c["plain"] > 0 and c["cross_channel"] > 0 and c["clamped"] > 0, c
        assert c["max_distance"] > 256, c  # beyond the row above: a plain distance across rows


def test_squeeze_stream_multiplier_is_the_widest_channel():
    """Squeeze leaves channels of several widths in one group stream: the special distances count in rows of the
    widest, and a copy 'from the row above' in a narrower channel only matches with that multiplier."""
    import synth
    w, h = 520, 300
    src = flat_picture(w, h, 3)
    f = synth.encode_modular(w, h, 3, rct=6, squeeze=1, tree_kind=1, source=src, lz77=2)
    c = synth.lz77_census()
    out, _ = oracle(f)
    assert np.array_equal(out, src) and c["special"] > 0


# ---- token-level frames: the model decodes forward, the writer adds copies to the tokens it was given -----------------
def run_chooser(seed):
    """Residuals toward a blocky target (runs of zeros, repeated rows) with a few random ones."""
    rng = np.random.default_rng(seed)

    def choose(guess, mul, x, y, c):
        if rng.random() < 0.02:
            return int(rng.integers(-3, 4))
        target = ((x // 24) * 37 + (y // 16) * 11 + 60 * c) % 256
        return M.clamp_dec((target - guess) // mul, mul)
    return choose


def multipliers(frame):
    """The widest channel of each section's stream (the unit of the special distances)."""
    nc = 1 if frame.grey else 3
    gd = 128 << frame.group_shift
    small = frame.w <= gd and frame.h <= gd
    _, rects, n_lf = M.section_layout(frame.w, frame.h, frame.group_shift, nc)
    m0 = max([frame.palette[0]] if frame.palette else [0])
    if small:
        m0 = max(m0, frame.w)
    return [m0] + [0] * n_lf + [r[2] for r in rects]


def token_case(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    tree = lambda depth=4, props=(0, 1, 3, 6, 9, 10), **kw: M.random_tree(rng, depth, list(props), **kw)  # noqa: E731
    if name == "ans_tree":
        return M.Frame(300, 260, tree(), group_shift=0)
    if name == "prefix_tree":
        return M.Frame(280, 150, tree(), group_shift=0, prefix=True, hybrid=(2, 1, 1))
    if name == "wp_tree":
        return M.Frame(200, 150, tree(4, [15, 0, 9, 14], leaf_preds=[6, 6, 5, 1]), group_shift=0)
    if name == "palette":
        return M.Frame(270, 140, tree(3, [0, 2, 5]), group_shift=0, palette=(40, M.index_chooser(3, 40)))
    if name == "local_rct_trees":
        groups = {g: {"rct": [(0, 6 + g)], "tree": tree(3, [0, 3, 10]) if g % 2 else None} for g in range(6)}
        return M.Frame(300, 200, tree(), group_shift=0, groups=groups, prefix=True)
    raise KeyError(name)


TOKEN_CASES = ["ans_tree", "prefix_tree", "wp_tree", "palette", "local_rct_trees"]
_TOK = {}


def token_frame(name, mode, fault=None, lz=None):
    """(model frame, written file) of a token case with LZ77 copies of `mode`."""
    import synth
    key = (name, mode, fault, str(lz))
    if key not in _TOK:
        if name not in _TOK:
            _TOK[name] = token_case(name).decode(run_chooser(sum(map(ord, name))))
        frame = _TOK[name]
        spec = dict(frame.spec)
        spec["lz77"] = dict(lz or {}, mode=mode, multipliers=multipliers(frame), fault=fault)
        _TOK[key] = (frame, synth.encode_modular_tokens(spec), synth.lz77_census())
    return _TOK[key]


def model_planes(frame):
    p = frame.planes
    return np.repeat(p, 3, axis=0) if p.shape[0] == 1 else p


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", TOKEN_CASES)
def test_token_frames_equal_the_model(name, mode):
    frame, data, census = token_frame(name, mode)
    out, planes = oracle(data)
    assert np.array_equal(planes.reshape(-1), model_planes(frame).reshape(-1).astype(np.int32))
    assert np.array_equal(out, frame.u8)
    assert census["copies"] > 0, census
    if mode == 2 and name != "palette":  # palette indices are random: few runs there
        assert census["special"] > 0 and census["plain"] > 0, census


def test_token_lz77_parameters():
    """Other min_symbol / min_length / length configurations than the writer's defaults."""
    frame, data, census = token_frame("ans_tree", 2, lz={"min_symbol": 100, "min_length": 7, "length": (2, 1, 0)})
    _, planes = oracle(data)
    assert np.array_equal(planes.reshape(-1), model_planes(frame).reshape(-1).astype(np.int32)) and census["copies"] > 0


# ---- a stream longer than the window ---------------------------------------------------------------------------------
def long_stream_frame():
    """2048 x 1024, group size 1024, one Zero leaf: two group streams of 3 x 1024^2 symbols. Channel 1 repeats channel 0
    (noise, no shorter repeat), so the only copies are at distance 2^20, one channel back."""
    import synth
    w, h = 2048, 1024
    rng = np.random.default_rng(5)
    planes = rng.integers(0, 256, (3, h, w)).astype(np.int64)
    planes[1] = planes[0]
    sections = [{"use_global_tree": True, "wp": None, "transforms": [], "tokens": None}, None]
    for g in range(2):
        vals = planes[:, :, g * 1024:(g + 1) * 1024].reshape(-1) * 2  # pack_signed of a non-negative value
        sections.append({"use_global_tree": True, "wp": None, "transforms": [],
                         "tokens": list(zip([0] * vals.size, vals.tolist()))})
    spec = {"width": w, "height": h, "group_shift": 3, "tree": [("leaf", 0, 0, 0, 0)], "sections": sections,
            "lz77": {"mode": 2, "multipliers": [0, 0, 1024, 1024]}}
    return planes, synth.encode_modular_tokens(spec), synth.lz77_census()


def test_copy_at_distance_two_to_the_twenty():
    planes, data, census = long_stream_frame()
    assert census["max_stream"] == 3 << 20 and census["max_distance"] == 1 << 20 and census["copies"] > 0
    _, got = oracle(data)
    assert np.array_equal(got, planes.astype(np.int32))


# ---- errors ----------------------------------------------------------------------------------------------------------
ERROR_LZ = {"min_symbol": 128}  # room in the 8-bit alphabet for the token of an overflowing length


@pytest.mark.parametrize("fault", [1, 2], ids=["copy_first", "length_overflow"])
def test_lz77_errors_are_refused(fault):
    frame, data, _ = token_frame("ans_tree", 2, fault=(fault, 4), lz=ERROR_LZ)
    with pytest.raises(abi.JxgError):
        oracle(data)
    _, good, _ = token_frame("ans_tree", 2, lz=ERROR_LZ)
    _, planes = oracle(good)
    assert np.array_equal(planes.reshape(-1), model_planes(frame).reshape(-1).astype(np.int32))
