"""XYB-encoded (lossy) Modular frames on the GPU (jxg_modular_batch_add_output): the device's Y, X, B channels are
bit-exact against the CPU checker and the synthetic writer's source; XYB_F32_PLANAR is bit-identical to a float32
evaluation of ConvertModularXYBToF32Stage; every RGB format and orientation is within the float64 output stage's
bounds; regions are byte-identical to the crop of the whole decode; lossless frames in the same batch are unchanged;
pool fills, a corrupt group stream and refusals behave as for lossless frames."""
import os

import numpy as np
import pytest

import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from tests import f64_pipeline as fp
from tests import oracle_binding as ob

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "jxl")
RGB_FORMATS = [abi.FORMAT_RGB_U8, abi.FORMAT_RGBA_U8, abi.FORMAT_RGB_F32, abi.FORMAT_RGB_U16, abi.FORMAT_RGB_F16]
ALL_FORMATS = RGB_FORMATS + [abi.FORMAT_XYB_F32_PLANAR]
CUSTOM_F16 = (0.0625, 0.25, 0.5)
SENTINEL = 0xA5
UNSUPPORTED, ARGUMENT = -2, -22


@pytest.fixture(scope="module")
def ctx():
    c = j.JxgContext(0)
    yield c
    c.close()


def bicycles():
    return open(os.path.join(GOLDEN, "bicycles.jxl"), "rb").read()


def xyb_file(w, h, seed, squeeze=1, **kw):
    return synth.encode_modular(w, h, seed, rct=0, squeeze=squeeze, xyb=kw)


def _geometry(fr, fmt, region):
    """(rows, width in pixels) of an output buffer."""
    if fmt == abi.FORMAT_XYB_F32_PLANAR:
        return 3 * fr.info.coded_height, fr.info.coded_width
    if region is not None:
        return region[3], region[2]
    return fr.height, fr.width


def _alloc(fr, fmt, region=None, pad=0, device=False):
    import torch
    rows, w = _geometry(fr, fmt, region)
    stride = w * abi.BYTES_PER_PIXEL[fmt] + pad
    t = torch.full((rows, stride), SENTINEL, dtype=torch.uint8)
    return (t.cuda() if device else t.pin_memory()), stride


def _samples(fr, fmt, buf, region=None):
    rows, w = _geometry(fr, fmt, region)
    a = buf.cpu().numpy()[:, :w * abi.BYTES_PER_PIXEL[fmt]].copy()
    if fmt == abi.FORMAT_XYB_F32_PLANAR:
        return a.view(np.float32).reshape(3, fr.info.coded_height, w)
    dt = {abi.FORMAT_RGB_F32: np.float32, abi.FORMAT_RGB_U16: np.uint16, abi.FORMAT_RGB_F16: np.uint16}.get(fmt, np.uint8)
    return a.view(dt).reshape(rows, w, -1)


def decode(ctx, items, planes=False, expect_error=False):
    """items: (data, fmt, region, pad, device); fmt None: jxg_modular_batch_add (RGB u8). Returns the sample arrays
    (and the read_planes taps, or the failure)."""
    frames = [j.ModularParsedFrame(d) for d, *_ in items]
    b = j.ModularBatch(ctx)
    bufs, taps, failure = [], [], None
    try:
        for fr, (_, fmt, region, pad, device) in zip(frames, items):
            buf, stride = _alloc(fr, abi.FORMAT_RGB_U8 if fmt is None else fmt, region, pad, device)
            bufs.append(buf)
            b.add(fr, buf.data_ptr(), stride, device, region, fmt)
        b.run()
        if expect_error:
            with pytest.raises(abi.JxgError):
                b.wait()
            failure = b.last_failure
        else:
            b.wait()
        if planes:
            taps = [b.read_planes(i) for i in range(len(frames))]
    finally:
        b.close()
    outs = [_samples(fr, abi.FORMAT_RGB_U8 if it[1] is None else it[1], buf, it[2])
            for fr, buf, it in zip(frames, bufs, items)]
    if expect_error:
        return outs, failure
    return (outs, taps) if planes else outs


def decode_each(ctx, items, planes=False):
    """Each item in a batch of its own: frames of one batch must share their inverse-transform structure."""
    res = [decode(ctx, [it], planes=planes) for it in items]
    if planes:
        return [r[0][0] for r in res], [r[1][0] for r in res]
    return [r[0] for r in res]


def convert_f32(planes, q):
    """ConvertModularXYBToF32Stage in float32 (each operation correctly rounded): X, Y, B planes."""
    y, x, b = (np.float32(p) for p in planes.astype(np.float32))
    sx, sy, sb = (np.float32(v) for v in q)
    return np.stack([x * sx, y * sy, (b + y) * sb]).astype(np.float32)


def expected(data, fmt):
    """(ref, mag, tf, orientation) for fp.check_output: stage C of the converted planes in float64."""
    fr = j.ModularParsedFrame(data)
    c = fr.colour(fmt)
    d = c["desc"]
    _, planes = ob.decode_modular_file(data, planes=True)
    import types
    f = types.SimpleNamespace(output_tf=int(d.output_tf), opsin_biases=np.array(list(d.opsin_biases), np.float64),
                              intensity_target=float(d.intensity_target), output_gamma=float(d.output_gamma),
                              output_luminances=np.array(list(d.output_luminances), np.float64),
                              opsin_inverse_matrix=np.array(list(d.opsin_inverse_matrix), np.float64).reshape(3, 3))
    ref, mag = fp.stage_c(f, convert_f32(planes, c["lf_quant"]).astype(np.float64))
    return ref, mag, int(d.output_tf), int(d.orientation)


def cases():
    return [("bicycles", bicycles()), ("squeeze", xyb_file(600, 520, 1)), ("flat", xyb_file(530, 300, 2, squeeze=0)),
            ("custom", xyb_file(400, 270, 3, lf_quant=CUSTOM_F16)), ("grey", xyb_file(300, 200, 4, colour=6))]


def test_read_planes_bit_exact(ctx):
    cs = cases()
    _, taps = decode_each(ctx, [(d, abi.FORMAT_RGB_U8, None, 0, False) for _, d in cs], planes=True)
    for (name, d), t in zip(cs, taps):
        _, want = ob.decode_modular_file(d, planes=True)
        assert np.array_equal(t, want), name
    assert np.array_equal(taps[1], synth.modular_xyb_source(600, 520, 1))
    assert np.array_equal(taps[3], synth.modular_xyb_source(400, 270, 3, CUSTOM_F16))


def test_xyb_planar_bit_identical(ctx):
    cs = cases()
    outs = decode_each(ctx, [(d, abi.FORMAT_XYB_F32_PLANAR, None, 4, dev) for (_, d), dev in zip(cs, (0, 1, 0, 1, 0))])
    for (name, d), g in zip(cs, outs):
        _, planes = ob.decode_modular_file(d, planes=True)
        want = convert_f32(planes, j.ModularParsedFrame(d).colour()["lf_quant"])
        assert np.array_equal(g.view(np.uint32), want.view(np.uint32)), name


@pytest.mark.parametrize("fmt", RGB_FORMATS)
def test_output_stage(ctx, fmt):
    """All orientations, every colour encoding the synthetic header reaches (sRGB, linear, gamma, PQ, HLG, BT.709,
    grey, DCI), custom factors and the fixture, against the float64 output stage."""
    files = [xyb_file(300, 180, 60 + o, squeeze=o % 2, orientation=o) for o in range(1, 9)]
    files += [xyb_file(260, 170, 70 + c, colour=c) for c in range(8)]
    files += [xyb_file(270, 150, 80, lf_quant=CUSTOM_F16, orientation=6), bicycles()]
    outs = decode_each(ctx, [(d, fmt, None, 0, False) for d in files])
    for i, (d, g) in enumerate(zip(files, outs)):
        ref, mag, tf, o = expected(d, fmt)
        fp.check_output(fmt, g, ref, mag, tf, o, what=f"case {i}")


def _crop(img, r):
    x, y, w, h = r
    return img[y:y + h, x:x + w]


@pytest.mark.parametrize("orientation", [1, 6])
def test_regions_are_crops_of_the_whole_decode(ctx, orientation):
    data = xyb_file(700, 530, 90 + orientation, orientation=orientation)
    fr = j.ModularParsedFrame(data)
    W, H = fr.width, fr.height
    regions = [(0, 0, W, H), (0, 0, 1, 1), (W - 1, H - 1, 1, 1), (W - 37, 0, 37, H), (0, H - 5, W, 5),
               (123, 77, 211, 190), (300, 260, 1, 1), (255, 255, 2, 2)]
    for fmt in (abi.FORMAT_RGB_U8, abi.FORMAT_RGB_F16, abi.FORMAT_RGBA_U8):
        whole = decode(ctx, [(data, fmt, None, 0, False)])[0]
        for device, pad in ((False, 0), (True, 0), (False, 8), (True, 12)):
            outs = decode(ctx, [(data, fmt, r, pad, device) for r in regions])
            for r, g in zip(regions, outs):
                assert g.tobytes() == np.ascontiguousarray(_crop(whole, r)).tobytes(), (fmt, r, device, pad)
    whole = decode(ctx, [(bicycles(), None, None, 0, False)])[0]
    bf = j.ModularParsedFrame(bicycles())
    regs = [(1000, 600, 24, 31), (0, 0, 1, 1), (511, 300, 257, 40)]
    outs = decode(ctx, [(bicycles(), None, r, 0, True) for r in regs])
    for r, g in zip(regs, outs):
        assert g.tobytes() == np.ascontiguousarray(_crop(whole, r)).tobytes(), r
    assert bf.width == 1024


def test_mixed_batches_with_lossless_frames(ctx):
    """Frames of one size with Squeeze (and RCT): the lossy frames' plans are the lossless plan or a prefix of it."""
    lossless = [synth.encode_modular(600, 520, 7, 6, 1, 2), synth.encode_modular(600, 520, 8, 6, 1, 1)]
    lossy = [xyb_file(600, 520, 11), synth.encode_modular(600, 520, 12, rct=6, squeeze=1, xyb={"colour": 6}),
             xyb_file(600, 520, 13, orientation=6)]
    items = [(lossless[0], None, None, 0, False), (lossy[0], abi.FORMAT_RGB_F32, None, 0, True),
             (lossless[1], abi.FORMAT_RGB_U8, None, 0, False), (lossy[1], abi.FORMAT_RGB_U16, (5, 7, 300, 200), 6, False),
             (lossless[0], None, (10, 20, 100, 90), 0, True), (lossy[2], None, None, 0, False)]
    for order in (items, items[::-1]):
        mixed = decode(ctx, order)
        alone = [decode(ctx, [it])[0] for it in order]
        for i, (a, b) in enumerate(zip(mixed, alone)):
            assert a.tobytes() == b.tobytes(), i
    mixed = decode(ctx, items)
    for k, i in ((0, 0), (1, 2)):
        assert np.array_equal(mixed[i], ob.decode_modular_file(lossless[k]))
    assert np.array_equal(mixed[4], _crop(ob.decode_modular_file(lossless[0]), (10, 20, 100, 90)))


@pytest.mark.parametrize("fill", [0xFF, 0x7F])
def test_pool_fills(ctx, fill):
    items = [(xyb_file(600, 520, 13), fmt, None, 0, False) for fmt in ALL_FORMATS]
    items += [(xyb_file(600, 520, 13), abi.FORMAT_RGB_U8, (100, 100, 300, 200), 0, True)]
    fresh = decode(ctx, items)
    ctx.set_pool_fill(fill)
    try:
        poisoned = decode(ctx, items)
    finally:
        ctx.set_pool_fill(-1)
    for a, b in zip(fresh, poisoned):
        assert a.tobytes() == b.tobytes()


def test_corrupt_group_stream_is_named(ctx):
    """Bytes changed inside the last group's section (a 512 x 512 frame has 2 x 2 groups, the last section ends the
    file): jxg_modular_batch_wait names that frame and group; the other frames of the batch still decode."""
    good = xyb_file(512, 512, 14)
    fr = j.ModularParsedFrame(good)
    corrupt = bytearray(good)
    at = len(good) - fr.info.hf_bytes // 8
    for k in range(16):
        corrupt[at + k] ^= 0x5A
    items = [(xyb_file(512, 512, 15), None, None, 0, False), (bytes(corrupt), abi.FORMAT_RGB_F32, None, 0, False)]
    outs, failure = decode(ctx, items, expect_error=True)
    assert failure == (1, 3), failure
    assert outs[0].tobytes() == decode(ctx, [items[0]])[0].tobytes()


def test_refusals_leave_the_batch_unchanged(ctx):
    import torch
    lossy = j.ModularParsedFrame(xyb_file(300, 200, 16))
    lossless = j.ModularParsedFrame(synth.encode_modular(300, 200, 7, 6, 1, 2))
    ref = decode(ctx, [(synth.encode_modular(300, 200, 7, 6, 1, 2), None, None, 0, False)])[0]
    b = j.ModularBatch(ctx)
    try:
        scratch = torch.zeros((800, 4096), dtype=torch.uint8).pin_memory()
        refusals = [(lossless, abi.FORMAT_RGB_F32, None, UNSUPPORTED), (lossless, abi.FORMAT_XYB_F32_PLANAR, None, UNSUPPORTED),
                    (lossy, 9, None, ARGUMENT), (lossy, abi.FORMAT_XYB_F32_PLANAR, (0, 0, 10, 10), ARGUMENT),
                    (lossy, abi.FORMAT_RGB_F32, (290, 0, 20, 10), ARGUMENT)]
        for fr, fmt, reg, code in refusals:
            with pytest.raises(abi.JxgError) as e:
                b.add(fr, scratch.data_ptr(), 4096, False, reg, fmt)
            assert e.value.code == code, (fmt, reg)
        with pytest.raises(abi.JxgError) as e:  # a stride too small for the f32 row
            b.add(lossy, scratch.data_ptr(), 300 * 12 - 4, False, None, abi.FORMAT_RGB_F32)
        assert e.value.code == -9
        assert b.lz77_stats() == {"lz77_streams": 0, "rle_streams": 0, "window_bytes": 0}
        out = torch.full((200, 900), SENTINEL, dtype=torch.uint8).pin_memory()
        b.add(lossless, out.data_ptr(), 900, False, None, abi.FORMAT_RGB_U8)
        b.run()
        b.wait()
        launches = b.stats()["kernel_launches"]
    finally:
        b.close()
    assert out.numpy().reshape(200, 300, 3).tobytes() == ref.tobytes()
    b = j.ModularBatch(ctx)
    try:
        out2 = torch.full((200, 900), SENTINEL, dtype=torch.uint8).pin_memory()
        b.add(lossless, out2.data_ptr(), 900, False)
        b.run()
        b.wait()
        assert b.stats()["kernel_launches"] == launches
    finally:
        b.close()


def test_decode_modular_files_formats(ctx):
    import torch
    files = [xyb_file(300, 200, 17, orientation=6), xyb_file(300, 200, 18)]
    for pf, fmt in ((j.JxlPixelFormat("RGB", "F16"), abi.FORMAT_RGB_F16), (j.JxlPixelFormat("RGBA", "U8"), abi.FORMAT_RGBA_U8),
                    (j.JxlPixelFormat(), abi.FORMAT_RGB_U8)):
        want = decode(ctx, [(d, fmt, None, 0, False) for d in files])
        for to_host in (True, False):
            got = j.decode_modular_files(ctx, files, to_host=to_host, pixel_format=pf)
            for g, w in zip(got, want):
                a = g.cpu()
                a = a.view(torch.uint16) if a.dtype == torch.float16 else a
                assert a.numpy().tobytes() == w.tobytes()
