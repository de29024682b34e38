"""Region decode on the GPU: a region frame stores the whole-frame GPU decode's bytes on the region, in every filter
configuration, orientation, entropy coding and format, host and device outputs, rows aligned or padded (the vector and
the scalar store paths of the fused filter kernel); mixed batches; the entropy work skipped; corrupt sections outside
and inside the selection; device padding; poisoned pools; the Python entry points."""
import ctypes as C

import numpy as np
import pytest

import jxl_rs_b200 as j
from jxl_rs_b200 import abi, decoder
from tests.test_region import FILTERS, FORMATS, _crops, _file, frame_halo_regions

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def ctx():
    c = j.JxgContext(0)
    yield c
    c.close()


def _stride(fmt, w, pad):
    """Rows of 64-byte multiples (vector stores allowed), or those plus a sample (scalar stores only)."""
    s = (w * abi.BYTES_PER_PIXEL[fmt] + 63) // 64 * 64
    return s + ((1 if fmt == abi.FORMAT_RGB_U8 else 4) if pad else 0)


def _view(fmt, a, w, h):
    bpp = abi.BYTES_PER_PIXEL[fmt]
    return np.ascontiguousarray(a[:, :w * bpp])


def _alloc(h, stride, device):
    import torch
    if device:
        return torch.full((h, stride), SENTINEL, dtype=torch.uint8, device="cuda")
    return torch.full((h, stride), SENTINEL, dtype=torch.uint8).pin_memory()


def _decode(ctx, items, fmt, device=False, pad=False, stats=None):
    """One batch of (parsed frame, region or None); returns each output's pixel bytes (h x w*bpp u8)."""
    b = j.Batch(ctx, len(items))
    bufs = []
    try:
        for pf, reg in items:
            w, h = (pf.width, pf.height) if reg is None else (reg[2], reg[3])
            stride = _stride(fmt, w, pad)
            buf = _alloc(h, stride, device)
            b.add(pf, buf.data_ptr(), stride, fmt, device, reg)
            bufs.append((buf, w, h))
        b.run()
        b.wait()
        if stats is not None:
            stats.update(b.entropy_stats())
    finally:
        b.close()
    out = []
    for buf, w, h in bufs:
        a = buf.cpu().numpy()
        if device:  # the row padding of a device buffer keeps the sentinel (a host buffer receives a copy of whole rows)
            assert (a[:, w * abi.BYTES_PER_PIXEL[fmt]:] == SENTINEL).all()
        out.append(_view(fmt, a, w, h))
    return out


def _crop(fmt, full, reg):
    x, y, w, h = reg
    bpp = abi.BYTES_PER_PIXEL[fmt]
    return full[y:y + h, x * bpp:(x + w) * bpp]


def _regions(pf, seed):
    """Random crops, regions at the filter halo of the first group line of each axis, and regions whose x and width are
    not multiples of 4 (per-sample stores on vector tiles)."""
    w, h = pf.width, pf.height
    return _crops(w, h, seed) + frame_halo_regions(pf, 1) + [(5, 7, min(203, w - 5), min(61, h - 7)), (w // 2 + 1, h // 3, min(66, w - w // 2 - 1), min(97, h - h // 3)),
                                 (70, 40, 130, 90)]


def _check_frame(ctx, pf, fmt, seed, device, pad):
    regs = _regions(pf, seed)
    full = _decode(ctx, [(pf, None)], fmt, device, pad)[0]
    outs = _decode(ctx, [(pf, r) for r in regs], fmt, device, pad)
    for r, o in zip(regs, outs):
        assert o.tobytes() == _crop(fmt, full, r).tobytes(), (fmt, r, device, pad)


@pytest.mark.parametrize("gab,epf", FILTERS)
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("pad", [False, True])
def test_region_equals_full_gpu_decode(ctx, gab, epf, device, pad):
    k = gab * 4 + epf
    for o in (1 + k % 8, 1 + (k + 3) % 8):
        pf = j.ParsedFrame(_file(700, 600, 20 + k, epf, gab, profile=3, entropy=k % 4, orientation=o, dist=1.5))
        _check_frame(ctx, pf, abi.FORMAT_RGB_U8, k * 10 + o, device, pad)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("pad", [False, True])
def test_region_formats(ctx, fmt, device, pad):
    for o in (1, 6):
        pf = j.ParsedFrame(_file(600, 520, 31, 2, 1, profile=1, orientation=o, dist=1.0))
        _check_frame(ctx, pf, fmt, fmt + o, device, pad)


def test_mixed_batch(ctx):
    """Region and whole frames in one batch across the lean (ANS), fast (prefix) and slow (LZ77) entropy kernels and
    several filter configurations, with several regions of one frame."""
    fmt = abi.FORMAT_RGB_U8
    pfs = [j.ParsedFrame(_file(700, 600, 40, 2, 1, entropy=0)), j.ParsedFrame(_file(600, 520, 41, 1, 0, entropy=1)),
           j.ParsedFrame(_file(520, 600, 42, 3, 1, entropy=2, orientation=5)), j.ParsedFrame(_file(640, 480, 43, 0, 1, entropy=3))]
    wholes = [_decode(ctx, [(pf, None)], fmt)[0] for pf in pfs]
    items = [(pfs[0], (10, 20, 224, 224)), (pfs[1], None), (pfs[0], (300, 250, 101, 77)), (pfs[2], (3, 5, 250, 300)),
             (pfs[3], None), (pfs[1], (255, 255, 2, 2)), (pfs[0], (0, 0, 700, 600)), (pfs[3], (400, 100, 240, 380))]
    st = {}
    outs = _decode(ctx, items, fmt, stats=st)
    assert st["lean"] and st["fast"] and st["slow"]
    for (pf, reg), o in zip(items, outs):
        w = wholes[pfs.index(pf)]
        assert o.tobytes() == (w if reg is None else _crop(fmt, w, reg)).tobytes(), reg
    plain = _decode(ctx, [(pfs[1], None), (pfs[3], None)], fmt)
    assert plain[0].tobytes() == outs[1].tobytes() and plain[1].tobytes() == outs[4].tobytes()


def test_streams_decoded_are_the_selected_groups(ctx):
    pf = j.ParsedFrame(_file(1000, 700, 50, 2, 1))
    regs = [(10, 10, 50, 50), (300, 300, 224, 224), (0, 0, 1000, 700)]
    want = 0
    for r in regs:
        d, _, _, _, n, _, _ = pf.region_desc(abi.FORMAT_RGB_U8, r)
        want += n // int(d.num_passes)
    st = {}
    _decode(ctx, [(pf, r) for r in regs], abi.FORMAT_RGB_U8, stats=st)
    assert st["lean"] + st["fast"] + st["slow"] == want < 2 * 12


def _add_region_desc(b, d, hf, off, ln, n, reg, buf, stride):
    lib = b._lib
    abi.check(lib, lib.jxg_batch_add_frame_region(b._h, C.byref(d), hf, off, ln, n, C.byref(abi.JxgRegion(*reg)),
                                                  C.c_void_p(buf.data_ptr()), stride, 0))


def test_corrupt_sections(ctx):
    """A corrupt section outside the region's groups does not touch the region; one inside fails with the frame's own
    group index; the whole decode fails either way."""
    import torch
    fmt = abi.FORMAT_RGB_U8
    pf = j.ParsedFrame(_file(1000, 700, 51, 2, 1))
    clean = _decode(ctx, [(pf, None)], fmt)[0]
    d, hf, off, ln, n = pf.desc(fmt)
    offs = np.ctypeslib.as_array(C.cast(off, C.POINTER(C.c_uint64)), shape=(n,)).copy()
    lens = np.ctypeslib.as_array(C.cast(ln, C.POINTER(C.c_uint32)), shape=(n,)).copy()
    size = int((offs + lens).max())
    def corrupt(g):
        data = np.frombuffer(C.string_at(hf.value, size), np.uint8).copy()
        data[offs[g]:offs[g] + lens[g]] = np.random.default_rng(g).integers(0, 256, int(lens[g]), dtype=np.uint8)
        return data

    reg = (320, 300, 100, 100)  # needs group (1, 1) = group 5 of the 4 x 3 grid, and nothing else
    bad0, bad5 = corrupt(0), corrupt(5)
    hp = bad0.ctypes.data
    stride = 100 * 3
    buf = torch.full((100, stride), SENTINEL, dtype=torch.uint8).pin_memory()
    b = j.Batch(ctx, 1)
    _add_region_desc(b, d, hp, off, ln, n, reg, buf, stride)
    b.run()
    b.wait()
    b.close()
    assert buf.numpy().tobytes() == _crop(fmt, clean, reg).tobytes()
    full = torch.empty((700, 3000), dtype=torch.uint8).pin_memory()
    b = j.Batch(ctx, 1)
    b.add_desc(d, hp, off, ln, n, full.data_ptr(), 3000, False)
    b.run()
    with pytest.raises(abi.JxgError):
        b.wait()
    b.close()
    # the corrupt group inside the selection: frame 1 of the batch, group 5 of the frame (group 0 of its sub-frame)
    buf2 = torch.full((100, stride), SENTINEL, dtype=torch.uint8).pin_memory()
    b = j.Batch(ctx, 2)
    _add_region_desc(b, d, hp, off, ln, n, reg, buf, stride)
    _add_region_desc(b, d, bad5.ctypes.data, off, ln, n, reg, buf2, stride)
    b.run()
    f, g = C.c_uint32(), C.c_uint32()
    r = b._lib.jxg_batch_wait(b._h, C.byref(f), C.byref(g))
    b.close()
    assert r != 0 and (f.value, g.value) == (1, 5)
    d2, _, _, _, n2, origin, _ = pf.region_desc(fmt, reg)
    assert n2 == 1 and origin == (256, 256)


def test_poisoned_pools(ctx):
    pf = j.ParsedFrame(_file(700, 600, 60, 2, 1, orientation=3))
    items = [(pf, r) for r in _regions(pf, 3)]
    try:
        ctx.set_pool_fill(0x00)
        a = _decode(ctx, items, abi.FORMAT_RGB_U8)
        ctx.set_pool_fill(0xFF)
        b = _decode(ctx, items, abi.FORMAT_RGB_U8)
    finally:
        ctx.set_pool_fill(-1)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_region_refused_with_xyb_and_taps(ctx):
    import torch
    pf = j.ParsedFrame(_file(600, 520, 31, 2, 1))
    buf = torch.empty((64, 4096), dtype=torch.uint8).pin_memory()
    b = j.Batch(ctx, 2)
    with pytest.raises(abi.JxgError):
        b.add(pf, buf.data_ptr(), 4096, abi.FORMAT_XYB_F32_PLANAR, False, (0, 0, 8, 8))
    b.add(pf, buf.data_ptr(), 4096, abi.FORMAT_RGB_U8, False, (0, 0, 8, 8))
    b.run()
    b.wait()
    out = np.zeros(16 << 20, np.int32)
    assert b._lib.jxg_batch_read_coeffs(b._h, 0, out.ctypes.data_as(C.c_void_p), out.size) == -22
    assert b._lib.jxg_batch_read_xyb(b._h, 0, 0, out.ctypes.data_as(C.c_void_p), out.size) == -22
    b.close()


def test_python_entry_points(ctx):
    files = [_file(700, 600, 20 + k, 2, 1, orientation=o) for k, o in ((0, 1), (1, 6))]
    regs = [(5, 7, 203, 61), None]
    pfs = [j.ParsedFrame(f) for f in files]
    wholes = [_decode(ctx, [(pf, None)], abi.FORMAT_RGB_U8, pad=True)[0] for pf in pfs]
    for to_host in (True, False):
        outs = decoder.decode_files(ctx, files, to_host=to_host, regions=regs)
        assert tuple(outs[0].shape) == (61, 203, 3) and tuple(outs[1].shape) == (pfs[1].height, pfs[1].width, 3)
        for o, w, r in zip(outs, wholes, regs):
            o = o.cpu().numpy().reshape(o.shape[0], -1)
            assert o.tobytes() == (w if r is None else _crop(abi.FORMAT_RGB_U8, w, r)).tobytes()
    import torch
    bufs = [torch.empty((61, 203 * 3), dtype=torch.uint8).pin_memory(),
            torch.empty((pfs[1].height, pfs[1].width * 3), dtype=torch.uint8).pin_memory()]
    dec = decoder.PipelinedDecoder(0, depth=2, workers=4)
    try:
        dec.decode(files, [(b.data_ptr(), b.shape[1]) for b in bufs], regions=regs)
    finally:
        dec.close()
    assert bufs[0].numpy().tobytes() == _crop(abi.FORMAT_RGB_U8, wholes[0], regs[0]).tobytes()
    assert bufs[1].numpy().tobytes() == wholes[1].tobytes()
