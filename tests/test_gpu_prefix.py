"""Prefix decode of VarDCT frames on the GPU (jxg_parse_file_prefix + jxg_batch_add_parsed): groups with some passes
against the CPU oracle fed the same passes, groups without a pass against the float64 Upsample8x, complete prefixes
byte-identical to the whole-file decode, mixed batches, pool fills, error reports and launch counts."""
import ctypes as C

import numpy as np
import pytest

import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from tests import oracle_binding as ob
from tests import prefix_ref as pr

pytestmark = pytest.mark.gpu

FORMATS = [abi.FORMAT_RGB_U8, abi.FORMAT_RGBA_U8, abi.FORMAT_RGB_F32, abi.FORMAT_XYB_F32_PLANAR, abi.FORMAT_RGB_U16,
           abi.FORMAT_RGB_F16]


@pytest.fixture(scope="module")
def ctx():
    c = j.JxgContext(0)
    yield c
    c.close()


def _alloc(fr, fmt, region=None):
    import torch
    if fmt == abi.FORMAT_XYB_F32_PLANAR:
        rows, w = 3 * fr.info.coded_height, fr.info.coded_width
    else:
        rows, w = (fr.height, fr.width) if region is None else (region[3], region[2])
    stride = w * abi.BYTES_PER_PIXEL[fmt]
    return torch.full((rows, stride), 0xA5, dtype=torch.uint8).pin_memory(), stride


def decode(ctx, items, fmt=abi.FORMAT_RGB_U8, stop=0, keep=False):
    """items: frames, or (frame, region) pairs. Returns (batch, host byte arrays): the batch waited for, open with
    `keep` (the caller closes it; a context has one live batch), else closed and replaced by its stats()."""
    b = j.Batch(ctx, len(items))
    if stop:
        b.set_debug_stop(stop)
    outs = []
    for it in items:
        fr, reg = it if isinstance(it, tuple) else (it, None)
        t, stride = _alloc(fr, fmt, reg)
        outs.append(t)
        b.add(fr, t.data_ptr(), stride, fmt, False, reg)
    b.run()
    b.wait()
    outs = [t.numpy().copy() for t in outs]
    if keep:
        return b, outs
    st = b.stats()
    b.close()
    return st, outs


def lf_planes(data):
    """The host front end's LF planes of a whole file, float32 (3, yb, xb)."""
    fr = j.ParsedFrame(data)
    d = fr.desc(abi.FORMAT_RGB_F32)[0]
    xb, yb = (d.width + 7) // 8, (d.height + 7) // 8
    return np.stack([np.ctypeslib.as_array(C.cast(d.lf[c], C.POINTER(C.c_float)), shape=(yb, xb)).copy() for c in range(3)])


def oracle_passes(data, k):
    """The oracle decode of a whole file restricted to its first k passes (the desc and the sections of passes
    0 .. k-1): per-group coefficients and the XYB planes after the transforms."""
    fr = j.ParsedFrame(data)
    d, hf, off, ln, n = fr.desc(abi.FORMAT_RGB_U8)
    g = fr.info.num_groups
    d.num_passes = k
    cw, ch = fr.info.coded_width, fr.info.coded_height
    taps = {"coeffs": np.zeros((g, 3, 65536), np.int32),
            "xyb_idct": np.zeros((3, (ch + 7) // 8 * 8, (cw + 7) // 8 * 8), np.float32),
            "xyb_filtered": np.zeros((3, ch, cw), np.float32)}
    t = ob.JxoTaps(taps["coeffs"].ctypes.data, taps["xyb_idct"].ctypes.data, taps["xyb_filtered"].ctypes.data)
    out = np.zeros((fr.height, fr.width, 3), np.uint8)
    bad = C.c_uint32()
    assert ob.load().jxo_decode_frame(C.byref(d), hf, off, ln, k * g, out.ctypes.data, out.strides[0], C.byref(t), 1,
                                      C.byref(bad)) == 0
    return taps


def groups_of(fr):
    xg = (fr.info.coded_width + 255) // 256
    return [(g % xg, g // xg) for g in range(fr.info.num_groups)]


_UPSAMPLED = {}


def upsample_expectation(data, weights=None):
    """float64 Upsample8x of every group, (3, rows, cols) of the padded planes, and a bound of its sums' magnitudes."""
    key = (data, None if weights is None else weights.tobytes())
    if key not in _UPSAMPLED:
        _UPSAMPLED[key] = _upsample_expectation(data, weights)
    return _UPSAMPLED[key]


def _upsample_expectation(data, weights):
    lf = lf_planes(data).astype(np.float64)
    k = pr.upsample8_kernel(pr.default_weights8() if weights is None else weights)
    yb, xb = lf.shape[1:]
    out = np.zeros((3, yb * 8, xb * 8))
    for c in range(3):
        for gy in range((yb + 31) // 32):
            for gx in range((xb + 31) // 32):
                u = pr.upsample_lf_group(lf[c], gx, gy, k)
                out[c, gy * 256:gy * 256 + u.shape[0], gx * 256:gx * 256 + u.shape[1]] = u
    return out, np.abs(lf).max() * np.abs(k).sum(axis=(2, 3)).max()


def check_partial(ctx, data, cut, weights=None):
    """Decode data[:cut]: coefficients bit-exact against the oracle with each group's passes, XYB after the transforms
    within 1e-3 of it, zero-pass groups within f32 rounding of the float64 Upsample8x. Returns the pass counts."""
    fr = j.PrefixParsedFrame(data[:cut])
    k = fr.passes
    b, _ = decode(ctx, [fr], stop=2, keep=True)
    coeffs, xyb = b.read_coeffs(0), b.read_xyb(0, 0)
    b.close()
    up, mag = upsample_expectation(data, weights)
    for gi, (gx, gy) in enumerate(groups_of(fr)):
        sl = (slice(None), slice(gy * 256, gy * 256 + 256), slice(gx * 256, gx * 256 + 256))
        if k[gi] == 0:
            assert not coeffs[gi].any()
            err = np.abs(xyb[sl] - up[sl]).max()
            assert err <= 25 * 2.0 ** -22 * mag + 1e-7, (gi, err)
    for kk in sorted(set(k.tolist()) - {0}):
        taps = oracle_passes(data, kk)
        for gi, (gx, gy) in enumerate(groups_of(fr)):
            if k[gi] != kk:
                continue
            assert np.array_equal(coeffs[gi], taps["coeffs"][gi]), gi
            sl = (slice(None), slice(gy * 256, gy * 256 + 256), slice(gx * 256, gx * 256 + 256))
            assert np.abs(xyb[sl] - taps["xyb_idct"][sl]).max() <= 1e-3, gi
    return k


def mid_cut(data):
    """A cut half way through the HF sections."""
    start = pr.prefix_start(data)
    return (start + len(data)) // 2


@pytest.mark.parametrize("case", ["lean", "fast", "slow-lz77", "progressive"])
def test_partial_passes_match_the_oracle(ctx, case):
    if case == "progressive":
        data = pr.fixture("progressive_ac.jxl")  # three passes with shifts: k_entropy
    else:
        entropy = {"lean": 0, "fast": 1, "slow-lz77": 2}[case]
        data = synth.encode_synthetic(1100, 700, 70 + entropy, entropy=entropy)
    fr = j.PrefixParsedFrame(data[:mid_cut(data)])
    b, _ = decode(ctx, [fr], keep=True)
    st = b.entropy_stats()
    b.close()
    kernel = {"lean": "lean", "fast": "fast", "slow-lz77": "slow", "progressive": "slow"}[case]
    assert st[kernel] == int((fr.passes > 0).sum()) and st["lean"] + st["fast"] + st["slow"] == st[kernel]
    k = check_partial(ctx, data, mid_cut(data))
    assert len(set(k.tolist())) > 1  # groups with different pass counts
    if case == "progressive":
        for cut in sorted(set(pr.hf_sections(data)[0].ravel().tolist()))[1::27]:  # cuts reaching k_g = 1 and 2
            check_partial(ctx, data, max(cut, pr.prefix_start(data)))


@pytest.mark.parametrize("w,h,custom", [(200, 600, False), (264, 264, False), (600, 520, True), (2100, 264, False)])
def test_zero_pass_groups_are_the_upsampled_lf(ctx, w, h, custom):
    """At the end of HfGlobal no group has a pass: every group is the float64 Upsample8x of the LF image. 200 wide:
    one group column (the right margin reads 0.0); 264: a last group column and row one LF sample wide / tall."""
    weights, header = None, None
    if custom:
        bits = (np.random.default_rng(3).uniform(-0.05, 0.3, 210)).astype(np.float16).view(np.uint16)
        weights, header = pr.f16_bits_to_float(bits), {"weights8": bits.tolist()}
    data = synth.encode_synthetic(w, h, 80 + w, header=header)
    k = check_partial(ctx, data, pr.prefix_start(data), weights)
    assert not k.any()


@pytest.mark.parametrize("fmt", FORMATS)
def test_complete_prefix_is_byte_identical(ctx, fmt):
    files = [synth.encode_synthetic(600, 400, 90 + o, orientation=o) for o in range(1, 9)]
    files += [pr.fixture("progressive_ac.jxl")]
    for data in files:
        _, (a, b) = decode(ctx, [j.ParsedFrame(data), j.PrefixParsedFrame(data)], fmt)
        assert np.array_equal(a, b)


def test_mixed_batches_give_each_frame_alone(ctx):
    d1 = synth.encode_synthetic(1100, 700, 101)
    d2 = pr.fixture("progressive_ac.jxl")
    d3 = synth.encode_synthetic(900, 600, 102, entropy=1)
    items = [j.PrefixParsedFrame(d1[:mid_cut(d1)]), j.ParsedFrame(d3), (j.ParsedFrame(d1), (100, 50, 300, 200)),
             j.PrefixParsedFrame(d2[:mid_cut(d2)]), j.PrefixParsedFrame(d3[:pr.prefix_start(d3)])]
    _, together = decode(ctx, items)
    for it, got in zip(items, together):
        _, (alone,) = decode(ctx, [it])
        assert np.array_equal(got, alone)


def test_pool_fill_does_not_change_the_output(ctx):
    data = pr.fixture("progressive_ac.jxl")
    d2 = synth.encode_synthetic(700, 600, 103)
    frames = [j.PrefixParsedFrame(data[:mid_cut(data)]), j.PrefixParsedFrame(d2[:mid_cut(d2)])]
    outs = []
    for byte in (0x00, 0xFF):
        ctx.set_pool_fill(byte)
        try:
            outs.append(decode(ctx, frames)[1])
            b, _ = decode(ctx, frames, stop=2, keep=True)
            outs.append([b.read_xyb(0, 0), b.read_xyb(1, 0), b.read_coeffs(0), b.read_coeffs(1)])
            b.close()
        finally:
            ctx.set_pool_fill(-1)
    for x, y in zip(outs[0] + outs[1], outs[2] + outs[3]):
        assert np.array_equal(x, y)


def test_corrupt_byte_in_a_used_section_is_reported(ctx):
    data = synth.encode_synthetic(1100, 700, 104)
    cut = mid_cut(data)
    off, ln = pr.hf_sections(data)
    k = pr.group_passes(off, ln, cut)
    g = int(np.flatnonzero(k)[-1])
    bad = bytearray(data[:cut])
    for i in range(int(off[0, g]) + 8, int(off[0, g] + ln[0, g]) - 4, 7):
        bad[i] ^= 0x5A
    fr = j.PrefixParsedFrame(bytes(bad))
    t, stride = _alloc(fr, abi.FORMAT_RGB_U8)
    b = j.Batch(ctx, 1)
    b.add(fr, t.data_ptr(), stride, abi.FORMAT_RGB_U8, False)
    b.run()
    with pytest.raises(abi.JxgError) as e:
        b.wait()
    assert f"group {g}" in str(e.value)
    status = b.stream_status(0)
    b.close()
    assert status[g] != 0 and not status[k == 0].any()


def test_launch_counts(ctx):
    data = synth.encode_synthetic(1100, 700, 105)
    whole, _ = decode(ctx, [j.ParsedFrame(data)])
    complete, _ = decode(ctx, [j.PrefixParsedFrame(data)])
    partial, _ = decode(ctx, [j.PrefixParsedFrame(data[:mid_cut(data)])])
    n = whole["kernel_launches"]
    assert complete["kernel_launches"] == n
    assert partial["kernel_launches"] == n + 1  # k_upsample_lf8


def test_decode_prefixes(ctx):
    data = synth.encode_synthetic(700, 500, 106)
    cut = mid_cut(data)
    (got,) = j.decode_prefixes(ctx, [data[:cut]])
    _, (want,) = decode(ctx, [j.PrefixParsedFrame(data[:cut])])
    assert np.array_equal(got.numpy().reshape(want.shape), want)
