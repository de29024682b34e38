"""GPU vs oracle on synthetic frames written by synth/ (all DCT sizes the writer emits, EPF 0..3,
Gaborish on/off, single- and multi-section frames, odd sizes)."""
import numpy as np
import pytest

from jxl_rs_b200 import abi

pytestmark = pytest.mark.gpu

CASES = [
    # w, h, seed, distance, epf, gab, profile, entropy (0 ANS, 1 prefix codes, 2 ANS + LZ77, 3 prefix codes + LZ77)
    (256, 256, 1000, 0.5, 2, 1, 1, 0),     # BASELINE config 1 geometry: one group, single TOC entry
    (8, 8, 1, 1.0, 2, 1, 0, 0),
    (263, 131, 2, 0.7, 1, 0, 1, 0),        # ragged edges
    (777, 513, 3, 0.5, 3, 1, 2, 0),        # EPF iters 3 + 64x64 family
    (1024, 512, 4, 0.3, 0, 1, 1, 0),       # no EPF, fine quantisation
    (1920, 1080, 3000, 0.5, 2, 1, 1, 0),   # BASELINE config 3 frame
    # SURVEY §8 a11: DCT128X128 ... DCT256X256 (types 21..26, the CTA-cooperative transform path)
    (1024, 768, 31, 0.5, 2, 1, 3, 0),
    (1300, 1100, 33, 0.4, 3, 0, 3, 0),     # ragged groups next to 256x256 varblocks, EPF 3 without Gaborish
    # SURVEY §8 a6: prefix-coded AC streams, >= 16 clusters, codes longer than the 8-bit root table
    (1024, 768, 32, 0.5, 2, 1, 1, 1),
    (777, 513, 34, 0.3, 1, 1, 3, 1),       # prefix codes + every transform family
    (256, 256, 35, 0.5, 2, 1, 0, 1),       # single-section frame, prefix codes
    # SURVEY §8 a4: LZ77 inside the HF streams (entropy_coding/decode.rs:286-330), ANS and prefix coded
    (1024, 768, 36, 0.5, 2, 1, 1, 2),
    (777, 513, 37, 0.5, 1, 1, 2, 3),
]


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


@pytest.mark.parametrize("case", CASES)
def test_synthetic_parity(ctx, case):
    import torch
    import jxl_rs_b200 as j
    import synth
    from tests import oracle_binding as ob
    w, h, seed, dist, epf, gab, prof, ent = case
    data = synth.encode_synthetic(w, h, seed, dist, epf, gab, prof, 0, ent)
    ref, taps = ob.decode_file(data, abi.FORMAT_RGB_U8, taps=True)
    fr = j.ParsedFrame(data)
    out = torch.empty((h, w, 3), dtype=torch.uint8).pin_memory()
    b = j.Batch(ctx, 1)
    b.add(fr, out.data_ptr(), w * 3, abi.FORMAT_RGB_U8, False)
    b.run()
    b.wait()
    assert np.array_equal(b.read_coeffs(0), taps["coeffs"])
    diff = np.abs(out.numpy().astype(np.int32) - ref.astype(np.int32))
    assert diff.max() <= 1
    b.close()
    xout = torch.empty((3, h, w), dtype=torch.float32).pin_memory()
    b = j.Batch(ctx, 1)
    b.add(fr, xout.data_ptr(), w * 4, abi.FORMAT_XYB_F32_PLANAR, False)
    b.run()
    b.wait()
    b.close()
    d = np.abs(xout.numpy() - taps["xyb_filtered"])
    assert np.all((d <= 1e-3) | (d <= 1e-3 * np.abs(taps["xyb_filtered"])))


@pytest.mark.parametrize("orientation", [2, 3, 4, 5, 6, 7, 8])
def test_orientation(ctx, orientation):
    """ImageMetadata.orientation through the store (render/save.rs): host and device outputs, RGB8 and RGBA8 / f32."""
    import jxl_rs_b200 as j
    import synth
    from tests import oracle_binding as ob
    data = synth.encode_synthetic(263, 131, 40 + orientation, 0.5, 2, 1, 1, orientation=orientation)
    ref, _ = ob.decode_file(data, abi.FORMAT_RGB_U8)
    for to_host in (True, False):
        out = j.decode_files(ctx, [data], to_host=to_host)[0].cpu().numpy()
        assert out.shape == ref.shape == ((263, 131, 3) if orientation >= 5 else (131, 263, 3))
        assert np.abs(out.astype(np.int16) - ref.astype(np.int16)).max() <= 1
    ref4, _ = ob.decode_file(data, abi.FORMAT_RGBA_U8)
    out4 = j.decode_files(ctx, [data], j.JxlPixelFormat("RGBA", "U8"))[0].numpy()
    assert np.abs(out4.astype(np.int16) - ref4.astype(np.int16)).max() <= 1
    reff, _ = ob.decode_file(data, abi.FORMAT_RGB_F32)
    outf = j.decode_files(ctx, [data], j.JxlPixelFormat("RGB", "F32"))[0].numpy()
    assert np.abs(outf - reff).max() <= 1e-3


@pytest.mark.parametrize("orientation,colour", [(1, 0), (6, 0), (1, 5), (1, 6)])
def test_sixteen_bit_output_samples(ctx, orientation, colour):
    """a17: U16 (convert.rs:717-786) and F16 (convert.rs:789-857, clamp ranges of PQ / HLG outputs frame/render.rs:746-750):
    every code between store(ref - b) and store(ref + b), ref the float64 stage C of the GPU's own filtered planes and b
    its f32 bound (tests/f64_pipeline.py); the oracle's codes must meet the same rule on its own planes. Interior
    tiles, edge tiles and the orientation post-pass all carry 6-byte pixels."""
    import synth
    import torch
    import jxl_rs_b200 as j
    from tests import f64_pipeline as fp
    from tests import oracle_binding as ob
    w, h = 333, 271
    data = synth.encode_synthetic(w, h, 77, 0.5, 2, 1, 1, orientation=orientation, colour=colour)
    fr = j.ParsedFrame(data)
    xyb = torch.empty((3, h, w), dtype=torch.float32).pin_memory()
    b = j.Batch(ctx, 1)
    b.add(fr, xyb.data_ptr(), w * 4, abi.FORMAT_XYB_F32_PLANAR, False)
    b.run()
    b.wait()
    b.close()
    _, taps = ob.decode_file(data, abi.FORMAT_RGB_F32, taps=True)
    for fmt, dt in ((abi.FORMAT_RGB_U16, torch.uint16), (abi.FORMAT_RGB_F16, torch.float16)):
        ref, _ = ob.decode_file(data, fmt)
        out = torch.empty((fr.height, fr.width, 3), dtype=dt).pin_memory()
        b = j.Batch(ctx, 1)
        b.add(fr, out.data_ptr(), fr.width * 6, fmt, False)
        b.run()
        b.wait()
        b.close()
        d = fp.Frame(fr.desc(fmt)[0])
        got = out.view(torch.int16).numpy().view(np.uint16)
        for codes, planes, who in ((got, xyb.numpy(), "GPU"), (ref, taps["xyb_filtered"], "oracle")):
            c, mc, allow, _ = fp.stage_c(d, planes.astype(np.float64), full=True)
            fp.check_output(fmt, codes, c, mc, d.output_tf, d.orientation, f"{who} format {fmt}",
                            allow if who == "oracle" else 0.0)


@pytest.mark.parametrize("colour", [1, 2, 3, 4, 5, 6, 7])
def test_output_colour_encodings(ctx, colour):
    """SURVEY §8 a16: linear, gamma, PQ (P3), HLG (BT2100), BT709 (custom primaries, DCI white), grey, DCI curve (E
    white): the device's curves (exp2f / log2f) against the oracle's restatement of the reference's rational
    approximations; u8 within 1 LSB, f32 within 1e-3."""
    import jxl_rs_b200 as j
    import synth
    from tests import oracle_binding as ob
    data = synth.encode_synthetic(520, 300, 50 + colour, 0.5, 2, 1, 1, colour=colour)
    ref, _ = ob.decode_file(data, abi.FORMAT_RGB_U8)
    out = j.decode_files(ctx, [data])[0].numpy()
    diff = np.abs(out.astype(np.int16) - ref.astype(np.int16))
    assert diff.max() <= 1 and (diff > 0).mean() < 0.02
    reff, _ = ob.decode_file(data, abi.FORMAT_RGB_F32)
    outf = j.decode_files(ctx, [data], j.JxlPixelFormat("RGB", "F32"))[0].numpy()
    d = np.abs(outf - reff)
    assert np.all((d <= 1e-3) | (d <= 1e-3 * np.abs(reff)))


def _frame_vs_oracle(ctx, data, threads=0, planes=True):
    """One frame through the C ABI against the oracle: coefficients bit-exact, filtered XYB planes within 1e-3,
    RGB u8 within 1 LSB (< 1 % of the samples off by one)."""
    import torch
    import jxl_rs_b200 as j
    from tests import oracle_binding as ob
    ref, taps = ob.decode_file(data, abi.FORMAT_RGB_U8, taps=planes, threads=threads)
    fr = j.ParsedFrame(data, max(1, threads))
    h, w = fr.height, fr.width
    out = torch.empty((h, w, 3), dtype=torch.uint8).pin_memory()
    b = j.Batch(ctx, 1)
    try:
        b.add(fr, out.data_ptr(), w * 3, abi.FORMAT_RGB_U8, False)
        b.run()
        b.wait()
        if planes:
            assert np.array_equal(b.read_coeffs(0), taps["coeffs"]), "AC coefficients are not bit-exact"
    finally:
        b.close()
    diff = np.abs(out.numpy().astype(np.int16) - ref.astype(np.int16))
    assert diff.max() <= 1, f"u8 output differs by {diff.max()} LSB"
    assert (diff > 0).mean() < 0.01
    if planes:
        xout = torch.empty((3, h, w), dtype=torch.float32).pin_memory()
        b = j.Batch(ctx, 1)
        try:
            b.add(fr, xout.data_ptr(), w * 4, abi.FORMAT_XYB_F32_PLANAR, False)
            b.run()
            b.wait()
        finally:
            b.close()
        d = np.abs(xout.numpy() - taps["xyb_filtered"])
        assert np.all((d <= 1e-3) | (d <= 1e-3 * np.abs(taps["xyb_filtered"])))
    return out.numpy()


def test_config2_frame_vs_oracle(ctx):
    """BASELINE config 2's own frame (3840x2160, seed 2000, distance 0.5, profile 1, EPF 2 — frame 0 of bench.py's
    batch) against the oracle, and the same frame inside a batch: position in the batch must not matter."""
    import jxl_rs_b200 as j
    import synth
    synth.set_threads(8)
    try:
        a = synth.encode_synthetic(3840, 2160, 2000, 0.5, 2, 1, 1)
        c = synth.encode_synthetic(3840, 2160, 2001, 0.5, 2, 1, 1)
    finally:
        synth.set_threads(1)
    alone = _frame_vs_oracle(ctx, a, threads=8)
    outs = j.decode_files(ctx, [a, c, a, c, a])
    assert np.array_equal(outs[0].numpy(), alone)
    assert np.array_equal(outs[0].numpy(), outs[2].numpy()) and np.array_equal(outs[0].numpy(), outs[4].numpy())
    assert np.array_equal(outs[1].numpy(), outs[3].numpy())
    assert not np.array_equal(outs[0].numpy(), outs[1].numpy())


def test_config3_batch_vs_oracle(ctx):
    """BASELINE config 3's shape (1920x1080 frames in one batch; 8 of the 64 per GPU, the oracle decodes each on the
    CPU): every frame of the batch against the oracle, u8 within 1 LSB."""
    import jxl_rs_b200 as j
    import synth
    from tests import oracle_binding as ob
    datas = [synth.encode_synthetic(1920, 1080, 3000 + i, 0.5, 2, 1, 1) for i in range(8)]
    outs = j.decode_files(ctx, datas)
    for d, o in zip(datas, outs):
        ref, _ = ob.decode_file(d, abi.FORMAT_RGB_U8, threads=8)
        diff = np.abs(o.numpy().astype(np.int16) - ref.astype(np.int16))
        assert diff.max() <= 1 and (diff > 0).mean() < 0.01


def test_config4_16k_epf3_vs_oracle(ctx):
    """BASELINE config 4: one 16384x16384 frame (4096 groups), EPF iters 3, LF groups decoded on several host threads
    (jxg_parse_file_mt); RGB u8 within 1 LSB of the oracle. The coefficient / plane taps are skipped at this size
    (3.2 GB each); the smaller EPF-3 cases above hold those."""
    import synth
    synth.set_threads(16)
    try:
        data = synth.encode_synthetic(16384, 16384, 4000, 0.5, 3, 1, 1)
    finally:
        synth.set_threads(1)
    _frame_vs_oracle(ctx, data, threads=16, planes=False)
