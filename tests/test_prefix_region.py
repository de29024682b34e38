"""Regions of prefix frames, host side (no GPU): the groups a region of a partly received file decodes, their pass
counts and the LF window of the upsampling (jxg_parsed_prefix_region_plan), against the cone a region of the whole file
takes (jxg_parsed_region_desc), and the regions that are refused."""
import numpy as np
import pytest

import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from tests import prefix_ref as pr
from tests.test_prefix import FIXTURES

ARGUMENT = -22  # JXG_ERR_ARGUMENT


def cuts(data):
    """End of HfGlobal, half way through the HF sections, whole."""
    start = pr.prefix_start(data)
    return [start, (start + len(data)) // 2, len(data)]


def regions(w, h):
    """Each corner, the interior, the whole image and 1x1 (output coordinates)."""
    rw, rh = min(w, 97), min(h, 61)
    return [(0, 0, rw, rh), (w - rw, 0, rw, rh), (0, h - rh, rw, rh), (w - rw, h - rh, rw, rh),
            (w // 2 - rw // 2, h // 2 - rh // 2, rw, rh), (0, 0, w, h), (w // 3, h // 2, 1, 1)]


def whole_file_cone(whole, region):
    """Whole-frame group indices of the sub-frame a region of the whole file decodes (sub-frame raster order), and the
    sub-frame's LF rectangle (x0, y0, x1, y1)."""
    d, _, _, _, _, origin, _ = whole.region_desc(abi.FORMAT_RGB_U8, region)
    xg = (whole.info.coded_width + 255) // 256
    gx0, gy0 = origin[0] // 256, origin[1] // 256
    sxg, syg = (d.width + 255) // 256, (d.height + 255) // 256
    groups = [(gy0 + y) * xg + gx0 + x for y in range(syg) for x in range(sxg)]
    bx0, by0 = origin[0] // 8, origin[1] // 8
    return groups, (bx0, by0, bx0 + (d.width + 7) // 8, by0 + (d.height + 7) // 8)


def check_plan(data):
    whole = j.ParsedFrame(data)
    xb, yb = (whole.info.coded_width + 7) // 8, (whole.info.coded_height + 7) // 8
    seen = set()
    for cut in cuts(data):
        fr = j.PrefixParsedFrame(data[:cut])
        k = fr.passes
        for reg in regions(fr.width, fr.height):
            groups, passes, win = fr.region_plan(reg)
            want, (x0, y0, x1, y1) = whole_file_cone(whole, reg)
            assert groups.tolist() == want, (cut, reg)
            assert np.array_equal(passes, k[groups]), (cut, reg)
            if (passes == 0).any():
                assert win == (max(x0 - 2, 0), max(y0 - 2, 0), min(x1 + 2, xb), min(y1 + 2, yb)), (cut, reg)
            else:
                assert win == (0, 0, 0, 0), (cut, reg)
            seen.add(bool((passes == 0).any()))
    return seen


@pytest.mark.parametrize("name", FIXTURES)
def test_cone_of_fixtures(name):
    check_plan(pr.fixture(name))


@pytest.mark.parametrize("o", range(1, 9))
def test_cone_of_oriented_frames(o):
    seen = check_plan(synth.encode_synthetic(700, 600, 120 + o, orientation=o))
    assert seen == {False, True}  # cones with and without a group that has no pass


def test_count_only_and_short_buffers():
    data = synth.encode_synthetic(700, 600, 130)
    fr = j.PrefixParsedFrame(data[:pr.prefix_start(data)])
    lib = abi.load_library()
    reg = abi.JxgRegion(0, 0, 700, 600)
    n = abi.C.c_uint32()
    assert lib.jxg_parsed_prefix_region_plan(fr._h, abi.C.byref(reg), None, None, 0, abi.C.byref(n), None) == 0
    assert n.value == fr.info.num_groups
    groups = np.zeros(n.value, np.uint32)
    assert lib.jxg_parsed_prefix_region_plan(fr._h, abi.C.byref(reg), groups.ctypes.data, None, n.value - 1,
                                             abi.C.byref(n), None) == ARGUMENT


def test_refusals():
    data = synth.encode_synthetic(600, 400, 131)
    fr = j.PrefixParsedFrame(data[:pr.prefix_start(data)])
    for reg in [(0, 0, 0, 5), (10, 10, 5, 0), (600, 0, 1, 1), (0, 400, 1, 1), (590, 0, 11, 1), (0, 0, 601, 400)]:
        with pytest.raises(abi.JxgError) as e:
            fr.region_plan(reg)
        assert e.value.code == ARGUMENT, reg
    whole = j.ParsedFrame(data)  # a whole-file handle is not a prefix frame
    with pytest.raises(abi.JxgError) as e:
        j.PrefixParsedFrame.region_plan(whole, (0, 0, 16, 16))
    assert e.value.code == ARGUMENT
