"""Regions of prefix frames on the GPU (jxg_parse_file_prefix + jxg_batch_add_parsed_region): a region stores the whole
prefix decode's bytes on its rectangle at every cut, filter configuration, orientation, format and store path; the
upsampled groups on the cone's edges read the frame's LF samples, mirrors and 0.0 margins; a cone whose groups all have
every pass decodes as a region of the whole file; only the cone is decoded; mixed batches; corrupt sections; pool fills;
decode_prefixes."""
import ctypes as C

import numpy as np
import pytest

import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from tests import prefix_ref as pr
from tests.test_gpu_prefix import decode as prefix_decode
from tests.test_gpu_region import SENTINEL, _alloc, _crop, _regions, _stride, _view
from tests.test_region import FILTERS, FORMATS, _file

pytestmark = pytest.mark.gpu
U8 = abi.FORMAT_RGB_U8


@pytest.fixture(scope="module")
def ctx():
    c = j.JxgContext(0)
    yield c
    c.close()


def _run(ctx, items, fmt=U8, device=False, pad=False):
    """One batch of (parsed frame, region or None): (pixel bytes of each output, stats(), entropy_stats())."""
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
        st, est = b.stats(), b.entropy_stats()
    finally:
        b.close()
    outs = []
    for buf, w, h in bufs:
        a = buf.cpu().numpy()
        if device:
            assert (a[:, w * abi.BYTES_PER_PIXEL[fmt]:] == SENTINEL).all()
        outs.append(_view(fmt, a, w, h))
    return outs, st, est


def _check(ctx, pf, regs, fmt=U8, device=False, pad=False):
    """Each region of pf equals the crop of pf's whole decode, with equal store alignment."""
    (full,), _, _ = _run(ctx, [(pf, None)], fmt, device, pad)
    outs, _, _ = _run(ctx, [(pf, r) for r in regs], fmt, device, pad)
    for r, o in zip(regs, outs):
        assert o.tobytes() == _crop(fmt, full, r).tobytes(), (fmt, r, device, pad)


def _cuts(data):
    """End of HfGlobal, half way through the HF sections, whole."""
    start = pr.prefix_start(data)
    return [start, (start + len(data)) // 2, len(data)]


@pytest.mark.parametrize("gab,epf", FILTERS)
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("pad", [False, True])
def test_region_equals_the_crop(ctx, gab, epf, device, pad):
    k = gab * 4 + epf
    for o in (1 + k % 8, 1 + (k + 3) % 8):
        data = _file(700, 600, 20 + k, epf, gab, profile=3, entropy=k % 4, orientation=o, dist=1.5)
        regs = _regions(j.ParsedFrame(data), k * 10 + o)  # the frame's geometry: a prefix handle has no descriptor
        for cut in _cuts(data):
            _check(ctx, j.PrefixParsedFrame(data[:cut]), regs, U8, device, pad)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("pad", [False, True])
def test_region_formats(ctx, fmt, device, pad):
    for o in (1, 6):
        data = _file(600, 520, 31, 2, 1, profile=1, orientation=o, dist=1.0)
        regs = _regions(j.ParsedFrame(data), fmt + o)
        for cut in _cuts(data)[:2]:
            _check(ctx, j.PrefixParsedFrame(data[:cut]), regs, fmt, device, pad)


def test_progressive_cuts(ctx):
    """Three passes with shifts: cones whose groups have 1 and 2 passes, next to groups with all three."""
    data = pr.fixture("progressive_ac.jxl")
    seen = set()
    whole = j.ParsedFrame(data)
    for cut in sorted(set(pr.hf_sections(data)[0].ravel().tolist()))[1::27]:
        pf = j.PrefixParsedFrame(data[:max(cut, pr.prefix_start(data))])
        regs = _regions(whole, cut % 97)
        for r in regs:
            seen.update(pf.region_plan(r)[1].tolist())
        _check(ctx, pf, regs)
    assert {1, 2} <= seen


def _edge_regions(pf, hh=8):
    """Per group: a small region in its middle (its cone is that group alone) and regions hugging each of its edges
    from inside, more than the filter halo away (coded = display coordinates, orientation 1)."""
    w, h = pf.info.coded_width, pf.info.coded_height
    out = []
    for gy in range((h + 255) // 256):
        for gx in range((w + 255) // 256):
            x0, y0 = gx * 256, gy * 256
            x1, y1 = min(w, x0 + 256), min(h, y0 + 256)
            cx, cy = (x0 + x1) // 2, (y0 + y1) // 2
            out.append((max(x0, cx - 8), max(y0, cy - 8), min(16, x1 - max(x0, cx - 8)), min(16, y1 - max(y0, cy - 8))))
            if x1 - x0 > 2 * hh + 4 and y1 - y0 > 2 * hh + 4:
                out += [(x0 + hh + 1, cy - 2, 3, 4), (x1 - hh - 4, cy - 2, 3, 4), (cx - 2, y0 + hh + 1, 4, 3),
                        (cx - 2, y1 - hh - 4, 4, 3)]
    return out


def _edge_cases(pf, regs):
    """(side, the neighbour outside the cone has a pass) of every zero-pass cone group on an interior cone edge."""
    k = pf.passes
    xg = (pf.info.coded_width + 255) // 256
    yg = len(k) // xg
    seen = set()
    for r in regs:
        groups, passes, _ = pf.region_plan(r)
        cone = set(groups.tolist())
        for g, p in zip(groups.tolist(), passes.tolist()):
            if p:
                continue
            gx, gy = g % xg, g // xg
            for side, nx, ny in (("left", gx - 1, gy), ("right", gx + 1, gy), ("top", gx, gy - 1), ("bottom", gx, gy + 1)):
                if 0 <= nx < xg and 0 <= ny < yg and ny * xg + nx not in cone:
                    seen.add((side, bool(k[ny * xg + nx])))
    return seen


@pytest.mark.parametrize("w,h,custom", [(200, 600, False), (264, 264, False), (2100, 264, False), (600, 520, True)])
def test_cone_edges(ctx, w, h, custom):
    """Zero-pass groups on the cone's edges: 200 wide has one group column (its right margin reads 0.0); 264x264 has
    a last group column one LF sample wide, so a cone of column 0 alone must read 0.0 where the whole frame does; the
    custom weights8 reach the kernel. Cuts at the end of HfGlobal and at the end of each group's section, so that the
    neighbours outside a cone have passes or none. Sections arrive in raster order, so a zero-pass group's right and
    bottom neighbours never have a pass."""
    header = None
    if custom:
        bits = np.random.default_rng(3).uniform(-0.05, 0.3, 210).astype(np.float16).view(np.uint16)
        header = {"weights8": bits.tolist()}
    data = synth.encode_synthetic(w, h, 140 + w, header=header)
    off, ln = pr.hf_sections(data)
    start = pr.prefix_start(data)
    cuts = sorted({start} | {int(e) for e in (off[0] + ln[0]).tolist() if e > start} - {len(data)})
    seen = set()
    for cut in cuts:
        pf = j.PrefixParsedFrame(data[:cut])
        regs = _edge_regions(pf)
        seen |= _edge_cases(pf, regs)
        _check(ctx, pf, regs)
    if (w, h) == (600, 520):
        assert {("left", True), ("left", False), ("top", True), ("top", False), ("right", False),
                ("bottom", False)} <= seen
    if (w, h) == (2100, 264):
        assert {("left", True), ("left", False), ("right", False), ("bottom", False)} <= seen
    if (w, h) == (264, 264):
        pf = j.PrefixParsedFrame(data[:start])
        assert pf.region_plan((100, 100, 20, 20))[0].tolist() == [0]


def _first_group_cut(data):
    """A cut at the end of group 0's (only) section: group 0 has its pass, the groups after it none."""
    off, ln = pr.hf_sections(data)
    assert off.shape[0] == 1
    return int(off[0, 0] + ln[0, 0])


def test_complete_cone_is_a_whole_file_region(ctx):
    data = synth.encode_synthetic(1100, 700, 150)
    cut = _first_group_cut(data)
    pf, whole = j.PrefixParsedFrame(data[:cut]), j.ParsedFrame(data)
    reg = (10, 10, 100, 100)
    groups, passes, win = pf.region_plan(reg)
    assert groups.tolist() == [0] and passes.tolist() == [1] and win == (0, 0, 0, 0) and not pf.passes[1:].any()
    (a,), sa, _ = _run(ctx, [(pf, reg)])
    (b,), sb, _ = _run(ctx, [(whole, reg)])
    assert a.tobytes() == b.tobytes()
    assert sa["kernel_launches"] == sb["kernel_launches"] and sa["h2d_bytes"] == sb["h2d_bytes"]
    # a cone with groups short of passes but none without one launches no k_upsample_lf8; a zero-pass group next
    # to an entropy-decoded one adds it
    prog = pr.fixture("progressive_ac.jxl")
    off = pr.hf_sections(prog)[0]
    ppf = j.PrefixParsedFrame(prog[:int(off[1].max())])  # pass 1 of every group but the last has arrived
    preg = (0, 0, 64, 64)
    assert 0 < ppf.region_plan(preg)[1].min() < 3
    _, sp, _ = _run(ctx, [(ppf, preg)])
    _, sw, _ = _run(ctx, [(j.ParsedFrame(prog), preg)])
    assert sp["kernel_launches"] == sw["kernel_launches"]
    reg2 = (200, 10, 100, 100)  # groups 0 (its pass) and 1 (none)
    assert pf.region_plan(reg2)[1].tolist() == [1, 0]
    _, s2, _ = _run(ctx, [(pf, reg2)])
    _, w2, _ = _run(ctx, [(whole, reg2)])
    assert s2["kernel_launches"] == w2["kernel_launches"] + 1


def test_only_the_cone_is_decoded(ctx):
    data = synth.encode_synthetic(1100, 700, 151)
    start = pr.prefix_start(data)
    pf = j.PrefixParsedFrame(data[:(start + len(data)) // 2])
    regs = [(10, 10, 50, 50), (300, 300, 224, 224), (520, 250, 300, 200), (0, 0, 1100, 700)]
    want = sum(int((pf.region_plan(r)[1] > 0).sum()) for r in regs)
    _, _, est = _run(ctx, [(pf, r) for r in regs])
    assert est["lean"] + est["fast"] + est["slow"] == want
    _, small, _ = _run(ctx, [(pf, (300, 300, 100, 100))])
    _, full, _ = _run(ctx, [(pf, None)])
    assert small["h2d_bytes"] < full["h2d_bytes"]


def test_mixed_batch(ctx):
    """Prefix regions, whole prefixes, whole-file regions, whole frames and overlapping regions of one prefix frame, on
    the lean (ANS), fast (prefix code) and slow (LZ77) entropy kernels: each frame equals its decode alone."""
    files = [_file(700, 600, 160, 2, 1, entropy=0), _file(600, 520, 161, 1, 0, entropy=1),
             _file(520, 600, 162, 3, 1, entropy=2, orientation=5)]
    pre = [j.PrefixParsedFrame(d[:_cuts(d)[1]]) for d in files]
    zero = j.PrefixParsedFrame(files[0][:pr.prefix_start(files[0])])
    whole = [j.ParsedFrame(d) for d in files]
    items = [(pre[0], (10, 20, 224, 224)), (pre[0], (100, 100, 300, 200)), (pre[1], None), (whole[2], (3, 5, 250, 300)),
             (pre[2], (200, 200, 250, 280)), (whole[1], None), (zero, (400, 300, 200, 200)), (pre[1], (255, 255, 2, 2)),
             (pre[0], (0, 0, 700, 600)), (zero, None)]
    together, _, est = _run(ctx, items)
    assert est["lean"] and est["fast"] and est["slow"]
    for it, got in zip(items, together):
        (alone,), _, _ = _run(ctx, [it])
        assert got.tobytes() == alone.tobytes(), it[1]


def _wait_code(b):
    f, g = C.c_uint32(), C.c_uint32()
    r = b._lib.jxg_batch_wait(b._h, C.byref(f), C.byref(g))
    return r, f.value, g.value


def test_corrupt_sections(ctx):
    """A corrupt used section inside the cone is reported with the whole frame's group index; one outside the cone, and
    the bytes of the section the cut falls in (not used: it has not arrived whole), leave the region unchanged."""
    import torch
    data = synth.encode_synthetic(1100, 700, 170)
    off, ln = pr.hf_sections(data)
    part = 8  # the cut falls inside group 8's section: groups 0 .. 7 have their pass, the others none
    cut = int(off[0, part] + ln[0, part] // 2)
    k = pr.group_passes(off, ln, cut)
    assert k[:part].all() and not k[part:].any()
    g_in = 6  # group (1, 1) of the 5 x 3 grid; the region sits in its middle, its cone is that group alone
    reg = (256 + 118, 256 + 118, 20, 20)
    pf = j.PrefixParsedFrame(data[:cut])
    assert pf.region_plan(reg)[0].tolist() == [g_in]
    (clean,), _, _ = _run(ctx, [(pf, reg)])

    def corrupt(lo, hi):
        bad = bytearray(data[:cut])
        for i in range(lo, hi, 7):
            bad[i] ^= 0x5A
        return j.PrefixParsedFrame(bytes(bad))

    outside = corrupt(int(off[0, 0]) + 8, int(off[0, 0] + ln[0, 0]) - 4)  # group 0, decoded by the whole prefix only
    unused = corrupt(int(off[0, part]), cut)
    for fr in (outside, unused):
        (got,), _, _ = _run(ctx, [(fr, reg)])
        assert got.tobytes() == clean.tobytes()
    inside = corrupt(int(off[0, g_in]) + 8, int(off[0, g_in] + ln[0, g_in]) - 4)
    bufs = [torch.full((20, 60), SENTINEL, dtype=torch.uint8).pin_memory() for _ in range(2)]
    b = j.Batch(ctx, 2)
    b.add(pf, bufs[0].data_ptr(), 60, U8, False, (0, 0, 20, 20))
    b.add(inside, bufs[1].data_ptr(), 60, U8, False, reg)
    b.run()
    r, f, g = _wait_code(b)
    b.close()
    assert r != 0 and (f, g) == (1, g_in)


def test_pool_fill_does_not_change_the_output(ctx):
    data = pr.fixture("progressive_ac.jxl")
    d2 = synth.encode_synthetic(700, 600, 171)
    items = [(j.PrefixParsedFrame(data[:_cuts(data)[1]]), (500, 300, 700, 500)),
             (j.PrefixParsedFrame(d2[:_cuts(d2)[1]]), (300, 200, 300, 300)),
             (j.PrefixParsedFrame(d2[:pr.prefix_start(d2)]), (250, 250, 200, 100))]
    outs = []
    try:
        for byte in (0x00, 0xFF):
            ctx.set_pool_fill(byte)
            outs.append(_run(ctx, items)[0])
    finally:
        ctx.set_pool_fill(-1)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(*outs))


def test_decode_prefixes_with_regions(ctx):
    files = [synth.encode_synthetic(700, 500, 172), synth.encode_synthetic(600, 400, 173, orientation=6)]
    cut = [f[:_cuts(f)[1]] for f in files]
    regs = [(5, 7, 203, 61), None]
    pfs = [j.PrefixParsedFrame(c) for c in cut]
    _, want = prefix_decode(ctx, list(zip(pfs, regs)))  # tight rows, as decode_prefixes allocates them
    for to_host in (True, False):
        got = j.decode_prefixes(ctx, cut, to_host=to_host, regions=regs)
        assert tuple(got[0].shape) == (61, 203, 3) and tuple(got[1].shape) == (pfs[1].height, pfs[1].width, 3)
        for g, w in zip(got, want):
            assert g.cpu().numpy().reshape(w.shape).tobytes() == w.tobytes()
    with pytest.raises(ValueError):
        j.decode_prefixes(ctx, cut, regions=[None])
