"""Prefix decode of VarDCT frames, host side (no GPU): which passes each HF group of a cut file decodes, the cuts that
are refused, and the constants and restatements the GPU tests compare against (tests/test_gpu_prefix.py)."""
import ctypes as C
import re

import numpy as np
import pytest

import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from tests import prefix_ref as pr

OUT_OF_BOUNDS, ARGUMENT = -3, -22  # JXG_ERR_OUT_OF_BOUNDS, JXG_ERR_ARGUMENT
INFO_FIELDS = ["width", "height", "num_groups", "num_passes", "encoding", "coded_width", "coded_height", "orientation"]
FIXTURES = ["progressive_ac.jxl", "has_permutation.jxl", "zoltan_tasi_unsplash.jxl"]


def boundary_cuts(off, ln, start, size):
    """Every HF section boundary of the file and one byte either side, at or after the shortest accepted prefix."""
    ends = set((off + ln).ravel().tolist()) | set(off.ravel().tolist())
    cuts = {c + d for c in ends for d in (-1, 0, 1)} | {start, size}
    return sorted(c for c in cuts if start <= c <= size)


@pytest.mark.parametrize("name", FIXTURES)
def test_group_passes_follow_check_group(name):
    data = pr.fixture(name)
    off, ln = pr.hf_sections(data)
    full = j.ParsedFrame(data).info
    start = pr.prefix_start(data)
    cuts = boundary_cuts(off, ln, start, len(data))
    if len(cuts) > 400:  # large fixtures: every boundary of the first and last sections, a spread in between
        cuts = cuts[:150] + cuts[150:-150:max(1, (len(cuts) - 300) // 100)] + cuts[-150:]
    seen = set()
    for cut in cuts:
        fr = j.PrefixParsedFrame(data[:cut])
        want = pr.group_passes(off, ln, cut)
        assert np.array_equal(fr.passes, want), cut
        used = sum(int(ln[p, g]) for g in range(ln.shape[1]) for p in range(want[g]))
        assert fr.info.hf_bytes == used
        assert [getattr(fr.info, k) for k in INFO_FIELDS] == [getattr(full, k) for k in INFO_FIELDS]
        seen.update(want.tolist())
    # the cuts reach groups with all passes and, unless the permuted TOC puts every first pass before HfGlobal's end,
    # groups without a pass
    assert full.num_passes in seen and (0 in seen) == bool(np.any(off[0] + ln[0] > start))


@pytest.mark.parametrize("name", FIXTURES)
def test_cuts_before_hf_global_end_are_out_of_bounds(name):
    data = pr.fixture(name)
    off, ln = pr.hf_sections(data)
    start = pr.prefix_start(data)
    assert start <= off.min() or name == "has_permutation.jxl"  # without permutation the HF sections follow HfGlobal
    for cut in (start - 1, start - 2, start // 2, 64):
        assert pr.prefix_code(data[:cut]) == OUT_OF_BOUNDS
    with pytest.raises(abi.JxgError) as e:
        j.PrefixParsedFrame(data[:start - 1])
    assert e.value.code == OUT_OF_BOUNDS and "jxg_lf_parse_file" in str(e.value)
    assert np.all(j.PrefixParsedFrame(data[:start]).passes == pr.group_passes(off, ln, start))


def test_cut_inside_lf_sections():
    data = synth.encode_synthetic(2100, 600, 61, profile=0)
    lo, hi = 1, len(data)
    while lo < hi:  # shortest prefix the thumbnail parse accepts: the end of the last LF group
        mid = (lo + hi) // 2
        try:
            j.LfParsedFrame(data[:mid])
            hi = mid
        except abi.JxgError:
            lo = mid + 1
    lf_end = lo
    start = pr.prefix_start(data)
    assert lf_end < start
    for cut in (lf_end - 1, lf_end, (lf_end + start) // 2, start - 1):
        assert pr.prefix_code(data[:cut]) == -3
    assert pr.prefix_code(data[:start]) == 0


@pytest.mark.parametrize("name", FIXTURES)
def test_complete_prefix_is_the_whole_frame(name):
    data = pr.fixture(name)
    full = j.ParsedFrame(data).info
    fr = j.PrefixParsedFrame(data)
    assert np.all(fr.passes == full.num_passes)
    assert [getattr(fr.info, k) for k in INFO_FIELDS + ["hf_bytes"]] == [getattr(full, k) for k in INFO_FIELDS + ["hf_bytes"]]


def test_refusals():
    data = synth.encode_synthetic(600, 400, 62)
    fr = j.PrefixParsedFrame(data[:pr.prefix_start(data)])
    with pytest.raises(abi.JxgError) as e:
        fr.desc(abi.FORMAT_RGB_U8)
    assert e.value.code == ARGUMENT
    with pytest.raises(abi.JxgError) as e:
        fr.region_desc(abi.FORMAT_RGB_U8, (0, 0, 16, 16))
    assert e.value.code == -22
    whole = j.ParsedFrame(data)  # a whole-file handle has no pass counts
    lib = abi.load_library()
    out = np.zeros(whole.info.num_groups, np.uint8)
    assert lib.jxg_parsed_group_passes(whole._h, out.ctypes.data, out.size) == -22
    assert lib.jxg_parsed_group_passes(fr._h, out.ctypes.data, out.size - 1) == -22
    # one section (one group, one pass): it must be whole
    one = synth.encode_synthetic(200, 120, 63)
    assert j.ParsedFrame(one).info.num_groups == 1
    assert pr.prefix_code(one[:-1]) == -3
    assert np.all(j.PrefixParsedFrame(one).passes == 1)
    # a container must be whole
    box = open(pr.FIXTURES + "/progressive_ac.jxl", "rb").read()
    assert box[:2] != b"\xff\x0a"
    assert pr.prefix_code(box[:len(box) - 100]) == -1
    assert pr.prefix_code(box) == 0


def test_default_weights_match_the_generated_table():
    src = open(pr.HERE + "/../jxl_rs_b200/csrc/host/upsample8_weights.inc").read()
    nums = [float(v) for v in re.findall(r"(-?\d+\.\d+)f", src)]
    assert len(nums) == 210
    assert np.array_equal(np.float32(nums), np.float32(pr.default_weights8()))


def test_kernel_expansion_is_symmetric_and_normalised():
    k = pr.upsample8_kernel(pr.default_weights8())
    assert np.allclose(k, k[::-1, :, ::-1, :]) and np.allclose(k, k[:, ::-1, :, ::-1])
    assert np.allclose(k.sum(axis=(2, 3)), 1.0, atol=2e-3)  # each output is a weighted mean of its 5x5 window


def mirrored_everywhere(lf, gx, gy, kernel):
    """Upsample8x over the LF plane mirrored at every edge: what the reference's loop gives where its row buffer is
    written."""
    pad = np.pad(lf, 2, mode="symmetric")  # mirror(-1) = 0, mirror(-2) = 1
    lh, lw = lf.shape
    xs, ys = min(32, lw - gx * 32), min(32, lh - gy * 32)
    out = np.zeros((ys * 8, xs * 8))
    for y in range(ys):
        for x in range(xs):
            w = pad[gy * 32 + y:gy * 32 + y + 5, gx * 32 + x:gx * 32 + x + 5]
            out[y * 8:y * 8 + 8, x * 8:x * 8 + 8] = np.clip(np.einsum("abkl,kl->ab", kernel, w), w.min(), w.max())
    return out


def test_upsample_restatement_edge_cases():
    """The reference's row buffer starts zeroed, and two margins are never written: the right margin of a frame one
    group wide, and the last column of the window of the group left of a one-sample-wide last group column. There the
    window reads 0.0 (the outputs of the last two, resp. the last, LF columns); everywhere else it mirrors."""
    rng = np.random.default_rng(1)
    k = pr.upsample8_kernel(pr.default_weights8())
    lf = rng.uniform(0.5, 1.0, (41, 25))  # one group column; a 9-sample-tall second group row
    for gy in (0, 1):
        got, mir = pr.upsample_lf_group(lf, 0, gy, k), mirrored_everywhere(lf, 0, gy, k)
        assert np.array_equal(got[:, :-16], mir[:, :-16])
        assert got[:, -16:].min() < mir[:, -16:].min()  # the zeros pull the edge down
    lf = rng.uniform(0.5, 1.0, (33, 33))  # last group column and last group row one sample wide / tall
    for gy in (0, 1):
        got, mir = pr.upsample_lf_group(lf, 0, gy, k), mirrored_everywhere(lf, 0, gy, k)
        assert np.array_equal(got[:, :-8], mir[:, :-8]) and not np.allclose(got[:, -8:], mir[:, -8:])
    for gx, gy in ((1, 0), (1, 1)):  # the one-sample-wide groups themselves mirror
        assert np.array_equal(pr.upsample_lf_group(lf, gx, gy, k), mirrored_everywhere(lf, gx, gy, k))
    lf = rng.uniform(0.5, 1.0, (70, 90))  # interior groups: mirrored rows, copied columns
    for gx, gy in ((0, 0), (1, 1), (2, 2)):
        assert np.array_equal(pr.upsample_lf_group(lf, gx, gy, k), mirrored_everywhere(lf, gx, gy, k))


def test_custom_weights_header_round_trip():
    w = (np.arange(210) % 7 + 1).astype(np.float16).view(np.uint16).tolist()
    a = synth.encode_synthetic(600, 400, 64)
    b = synth.encode_synthetic(600, 400, 64, header={"weights8": w})
    assert a != b and len(b) > len(a)
    assert j.ParsedFrame(b).info.hf_bytes == j.ParsedFrame(a).info.hf_bytes
    assert synth.encode_synthetic(600, 400, 64, header=None) == a
