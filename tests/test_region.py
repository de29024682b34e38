"""Region decode on the CPU: the sub-frame jxg_parsed_region_desc slices out of a VarDCT frame, checked against a
brute-force restatement of the group selection, and decoded by the CPU oracle, which must give the whole-frame
decode's pixels on the region byte for byte."""
import ctypes as C
import functools
import os

import numpy as np
import pytest

import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from tests import oracle_binding as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "jxl")
FILTERS = [(gab, epf) for gab in (0, 1) for epf in range(4)]
FORMATS = [abi.FORMAT_RGB_U8, abi.FORMAT_RGBA_U8, abi.FORMAT_RGB_F32, abi.FORMAT_RGB_U16, abi.FORMAT_RGB_F16]


def display_pixel(o, w, h, x, y):
    """Display position of coded pixel (x, y) of a coded w x h image (the orientation pass, kernels.cu k_orient)."""
    return {1: (x, y), 2: (w - 1 - x, y), 3: (w - 1 - x, h - 1 - y), 4: (x, h - 1 - y), 5: (y, x), 6: (h - 1 - y, x),
            7: (h - 1 - y, w - 1 - x), 8: (y, w - 1 - x)}[o]


def halo(gab, epf):
    return (1 if gab else 0) + (2 if epf >= 1 else 0) + (1 if epf >= 2 else 0) + (3 if epf >= 3 else 0)


@functools.lru_cache(maxsize=2)
def _grid(w, h):
    ys, xs = np.mgrid[0:h, 0:w].astype(np.int32)
    return ys, xs


def restated_selection(w, h, gab, epf, o, region):
    """Brute force: the coded pixels whose display position lies in the region (searched over the whole image), the
    pixels they depend on (within the halo; with Gaborish + EPF 2 within the halo of every 64x32 tile that meets them),
    and every 256x256 group holding one of those. Returns (origin, size, groups of the sub-frame in raster order,
    coded window)."""
    rx, ry, rw, rh = region
    ys, xs = _grid(w, h)
    dx, dy = display_pixel(o, w, h, xs, ys)
    inside = (dx >= rx) & (dx < rx + rw) & (dy >= ry) & (dy < ry + rh)
    cols, rows = np.nonzero(inside.any(axis=0))[0], np.nonzero(inside.any(axis=1))[0]
    x0, x1, y0, y1 = int(cols[0]), int(cols[-1]) + 1, int(rows[0]), int(rows[-1]) + 1
    assert inside.sum() == rw * rh == (x1 - x0) * (y1 - y0)
    dep = (x0, x1, y0, y1)
    if gab and epf == 2:
        tiles = [(tx, ty) for ty in range(0, h, 32) for tx in range(0, w, 64)
                 if tx < x1 and tx + 64 > x0 and ty < y1 and ty + 32 > y0]
        dep = (min(t[0] for t in tiles), min(max(t[0] + 64 for t in tiles), w),
               min(t[1] for t in tiles), min(max(t[1] + 32 for t in tiles), h))
    hh = halo(gab, epf)
    xg, yg = (w + 255) // 256, (h + 255) // 256
    need = [(gx, gy) for gy in range(yg) for gx in range(xg)
            if gx * 256 <= dep[1] - 1 + hh and min(w, gx * 256 + 256) - 1 >= dep[0] - hh
            and gy * 256 <= dep[3] - 1 + hh and min(h, gy * 256 + 256) - 1 >= dep[2] - hh]
    gx0, gx1 = min(g[0] for g in need), max(g[0] for g in need) + 1
    gy0, gy1 = min(g[1] for g in need), max(g[1] for g in need) + 1
    origin = (gx0 * 256, gy0 * 256)
    size = (min(w, gx1 * 256) - origin[0], min(h, gy1 * 256) - origin[1])
    groups = [gy * xg + gx for gy in range(gy0, gy1) for gx in range(gx0, gx1)]
    return origin, size, groups, (x0 - origin[0], y0 - origin[1], x1 - x0, y1 - y0)


def regions_for(w, h, gab, epf):
    """Corners, 1x1, the whole image, regions on the image border, and regions whose edge lies within the halo of a
    group line on either side (display coordinates of a w x h output)."""
    hh = max(halo(gab, epf), 1)
    out = [(0, 0, w, h), (0, 0, 1, 1), (w - 1, h - 1, 1, 1), (w - 1, 0, 1, 1), (0, h - 1, 1, 1),
           (0, 0, min(w, 37), min(h, 29)), (w - min(w, 50), h - min(h, 41), min(w, 50), min(h, 41)),
           (0, h // 3, w, 1), (w // 2, 0, 1, h)]
    for line in (256, 512):
        for d in (-hh - 1, -hh, -1, 0, hh - 1, hh):
            x = line + d
            if 0 <= x < w - 3 and 0 <= x < h - 3:
                out.append((x, max(0, h // 2 - 10), 3, min(20, h - max(0, h // 2 - 10))))  # left edge near a group line
                out.append((max(0, w // 2 - 10), x, min(20, w - max(0, w // 2 - 10)), 3))  # top edge
                if x >= 8:
                    out.append((x - 8, x - 8, 8, 8))  # right / bottom edges just below x
    return out


def halo_regions(cw, ch, o, hh, max_lines=2):
    """Regions (display coordinates) whose edge sits just inside or just outside the filter halo of a group line, on
    both sides of each of the first `max_lines` coded group lines of each axis: a left / top edge at line + d and a
    right / bottom edge at line - 1 - d, d = hh - 1 (the group across the line is needed), hh and hh + 1 (it is not
    needed for the region's own pixels), and corners near two lines at once. The lines are taken in coded coordinates
    and the regions mapped through the orientation, so that flipped and transposed frames test their own lines."""
    coded = []
    xl, yl = list(range(256, cw, 256))[:max_lines], list(range(256, ch, 256))[:max_lines]
    ds = [d for d in (hh - 1, hh, hh + 1) if d >= 0]
    my, mx = max(0, ch // 2 - 32), max(0, cw // 2 - 32)
    for L in xl:
        for d in ds:
            coded += [(L + d, my, 5, min(64, ch - my)), (L - 1 - d - 4, my, 5, min(64, ch - my))]
    for L in yl:
        for d in ds:
            coded += [(mx, L + d, min(64, cw - mx), 5), (mx, L - 1 - d - 4, min(64, cw - mx), 5)]
    for Lx in xl[:1]:
        for Ly in yl[:1]:
            for d in ds:
                coded += [(Lx + d, Ly + d, 5, 5), (Lx - 1 - d - 4, Ly - 1 - d - 4, 5, 5)]
    out = []
    for x, y, w, h in coded:
        if x < 0 or y < 0 or x + w > cw or y + h > ch:
            continue
        a, b = display_pixel(o, cw, ch, x, y), display_pixel(o, cw, ch, x + w - 1, y + h - 1)
        out.append((min(a[0], b[0]), min(a[1], b[1]), abs(a[0] - b[0]) + 1, abs(a[1] - b[1]) + 1))
    return out


def frame_halo_regions(pf, max_lines=2):
    """halo_regions of a parsed frame (its coded size, orientation and filter halo)."""
    d = pf.desc(abi.FORMAT_RGB_U8)[0]
    return halo_regions(int(d.width), int(d.height), int(d.orientation) or 1, halo(int(d.gab), min(int(d.epf_iters), 3)),
                        max_lines)


@functools.lru_cache(maxsize=None)
def _file(w, h, seed, epf, gab, profile=0, entropy=0, orientation=1, dist=3.0):
    synth.set_threads(8)
    try:
        return synth.encode_synthetic(w, h, seed, dist, epf, gab, profile, entropy=entropy, orientation=orientation)
    finally:
        synth.set_threads(1)


def _arr(ptr, n, ctype):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape=(n,)).copy()


def _check_selection(pf, gab, epf, o, region):
    d0, _, off0, ln0, n0 = pf.desc(abi.FORMAT_RGB_U8)
    cw, ch = int(d0.width), int(d0.height)
    d, _, off, ln, n, origin, window = pf.region_desc(abi.FORMAT_RGB_U8, region)
    r_origin, r_size, groups, cwin = restated_selection(cw, ch, gab, epf, o, region)
    assert origin == r_origin and (int(d.width), int(d.height)) == r_size, (region, origin, r_origin)
    full_off, full_len = _arr(off0.value, n0, C.c_uint64), _arr(ln0.value, n0, C.c_uint32)
    G, P = n0 // int(d0.num_passes), int(d0.num_passes)
    want = [p * G + g for p in range(P) for g in groups]
    assert n == len(want)
    assert np.array_equal(_arr(off.value, n, C.c_uint64), full_off[want])
    assert np.array_equal(_arr(ln.value, n, C.c_uint32), full_len[want])
    # the window: display position of the coded window inside the sub-frame's display output
    sw, sh = r_size
    corners = [display_pixel(o, sw, sh, cwin[0] + a, cwin[1] + b) for a in (0, cwin[2] - 1) for b in (0, cwin[3] - 1)]
    assert window == (min(c[0] for c in corners), min(c[1] for c in corners))


SIZES = [(257, 131), (1000, 700)]


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("gab,epf", FILTERS)
@pytest.mark.parametrize("orientation", range(1, 9))
def test_group_selection_matches_restatement(size, gab, epf, orientation):
    w, h = size
    pf = j.ParsedFrame(_file(w, h, 5, epf, gab, orientation=orientation))
    dw, dh = pf.width, pf.height
    for region in regions_for(dw, dh, gab, epf) + frame_halo_regions(pf):
        _check_selection(pf, gab, epf, orientation, region)


@pytest.mark.parametrize("gab,epf", FILTERS)
def test_group_selection_4k(gab, epf):
    """3840x2160: every filter configuration, each at two orientations (all eight orientations are covered), with the
    regions of regions_for and regions at the halo of the first two group lines of each axis."""
    k = gab * 4 + epf
    for orientation in (1 + k, 1 + (k + 4) % 8):
        pf = j.ParsedFrame(_file(3840, 2160, 6, epf, gab, orientation=orientation, dist=8.0))
        for region in regions_for(pf.width, pf.height, gab, epf) + frame_halo_regions(pf):
            _check_selection(pf, gab, epf, orientation, region)


def _out(fmt, w, h):
    dt = {abi.FORMAT_RGB_F32: np.float32, abi.FORMAT_RGB_U16: np.uint16, abi.FORMAT_RGB_F16: np.float16}.get(fmt, np.uint8)
    return np.zeros((h, w, 4 if fmt == abi.FORMAT_RGBA_U8 else 3), dt)


def _oracle(d, hf, off, ln, n, w, h, fmt):
    out = _out(fmt, w, h)
    bad = C.c_uint32()
    r = ob.load().jxo_decode_frame(C.byref(d), hf, off, ln, n, out.ctypes.data, out.strides[0], None, 0, C.byref(bad))
    assert r == 0, r
    return out


def _check_exact(pf, fmt, regions):
    d, hf, off, ln, n = pf.desc(fmt)
    full = _oracle(d, hf, off, ln, n, pf.width, pf.height, fmt)
    for (x, y, w, h) in regions:
        sd, shf, soff, sln, sn, _, (wx, wy) = pf.region_desc(fmt, (x, y, w, h))
        o = int(sd.orientation) or 1
        dw, dh = (int(sd.height), int(sd.width)) if o >= 5 else (int(sd.width), int(sd.height))
        sub = _oracle(sd, shf, soff, sln, sn, dw, dh, fmt)
        got, want = sub[wy:wy + h, wx:wx + w], full[y:y + h, x:x + w]
        assert got.tobytes() == want.tobytes(), (fmt, (x, y, w, h))


def _crops(w, h, seed):
    rng = np.random.default_rng(seed)
    out = [(0, 0, w, h), (w - 1, h - 1, 1, 1), (1, 3, min(w - 1, 70), min(h - 3, 45))]
    for _ in range(3):
        cw, ch = int(rng.integers(1, min(w, 300) + 1)), int(rng.integers(1, min(h, 300) + 1))
        out.append((int(rng.integers(0, w - cw + 1)), int(rng.integers(0, h - ch + 1)), cw, ch))
    return out


@pytest.mark.parametrize("gab,epf", FILTERS)
def test_oracle_sub_frame_is_exact(gab, epf):
    """Synthetic frames of every filter configuration, profile 3 (DCT128 / DCT256 families), the four entropy codings
    and all eight orientations: the sub-frame decode equals the whole decode on the region, also for regions whose edge
    sits one pixel inside or outside the filter halo of a group line."""
    k = gab * 4 + epf
    for o in (1 + k % 8, 1 + (k + 3) % 8):
        pf = j.ParsedFrame(_file(700, 600, 20 + k, epf, gab, profile=3, entropy=k % 4, orientation=o, dist=1.5))
        _check_exact(pf, abi.FORMAT_RGB_U8, _crops(pf.width, pf.height, k * 10 + o) + frame_halo_regions(pf, 3)
                     + regions_for(pf.width, pf.height, gab, epf))


@pytest.mark.parametrize("fmt", FORMATS)
def test_oracle_sub_frame_formats(fmt):
    pf = j.ParsedFrame(_file(600, 520, 31, 2, 1, profile=1, orientation=6 if fmt % 2 else 1, dist=1.0))
    _check_exact(pf, fmt, _crops(pf.width, pf.height, fmt) + frame_halo_regions(pf, 1))


@pytest.mark.parametrize("name", ["zoltan_tasi_unsplash", "progressive_ac", "has_permutation", "grayscale",
                                  "opsin_inverse"])
def test_oracle_sub_frame_fixtures(name):
    pf = j.ParsedFrame(open(os.path.join(GOLDEN, name + ".jxl"), "rb").read())
    _check_exact(pf, abi.FORMAT_RGB_U8, _crops(pf.width, pf.height, len(name)) + frame_halo_regions(pf))


def test_whole_image_region_is_the_frame():
    pf = j.ParsedFrame(open(os.path.join(GOLDEN, "progressive_ac.jxl"), "rb").read())
    d, hf, off, ln, n = pf.desc(abi.FORMAT_RGB_U8)
    sd, shf, soff, sln, sn, origin, window = pf.region_desc(abi.FORMAT_RGB_U8, (0, 0, pf.width, pf.height))
    assert origin == (0, 0) and window == (0, 0) and sn == n and shf.value == hf.value
    assert np.array_equal(_arr(soff.value, sn, C.c_uint64), _arr(off.value, n, C.c_uint64))
    assert np.array_equal(_arr(sln.value, sn, C.c_uint32), _arr(ln.value, n, C.c_uint32))
    skip = {"lf", "transform_map", "raw_quant_map", "epf_map", "quant_lf", "ytox_map", "ytob_map"}
    for name, _ in abi.JxgFrameDesc._fields_:
        if name not in skip:
            a, b = getattr(d, name), getattr(sd, name)
            if name == "passes":
                a, b = C.cast(a, C.c_void_p).value, C.cast(b, C.c_void_p).value
            assert (list(a) == list(b)) if hasattr(a, "__len__") else a == b, name
    nb = ((int(d.width) + 7) // 8) * ((int(d.height) + 7) // 8)
    for name, ct in (("transform_map", C.c_uint8), ("raw_quant_map", C.c_int32), ("epf_map", C.c_uint8), ("quant_lf", C.c_uint8)):
        assert np.array_equal(_arr(getattr(d, name), nb, ct), _arr(getattr(sd, name), nb, ct)), name
    for c in range(3):
        assert np.array_equal(_arr(d.lf[c], nb, C.c_float), _arr(sd.lf[c], nb, C.c_float))


@pytest.mark.parametrize("region,fmt", [((0, 0, 0, 5), abi.FORMAT_RGB_U8), ((0, 0, 5, 0), abi.FORMAT_RGB_U8),
                                        ((250, 0, 8, 8), abi.FORMAT_RGB_U8), ((0, 0, 258, 1), abi.FORMAT_RGB_U8),
                                        ((0, 130, 1, 2), abi.FORMAT_RGB_U8), ((2 ** 32 - 1, 0, 2, 1), abi.FORMAT_RGB_U8),
                                        ((0, 0, 8, 8), abi.FORMAT_XYB_F32_PLANAR)])
def test_region_refusals(region, fmt):
    pf = j.ParsedFrame(_file(257, 131, 5, 2, 1))
    with pytest.raises(abi.JxgError) as e:
        pf.region_desc(fmt, region)
    assert e.value.code == -22  # JXG_ERR_ARGUMENT
