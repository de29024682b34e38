"""GPU Modular path (SURVEY §8 a18 / a19, BASELINE config 5) vs the CPU oracle: bit-exact i32 planes and u8 pixels
on synthetic lossless frames (RCT / Squeeze / three MA-tree kinds, ragged sizes), on the reference's real Modular
fixtures, and lossless round trips at full group counts."""
import os

import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests.gpu_modular import gpu_decode

pytestmark = pytest.mark.gpu

CASES = [
    # w, h, seed, rct, squeeze, tree_kind
    (64, 48, 1, 0, 0, 0),        # one group: everything is host-side section 0 (device path only stores)
    (300, 260, 2, 6, 0, 1),      # 2x2 groups, property tree
    (700, 530, 3, 6, 0, 2),      # weighted predictor
    (513, 300, 4, 0, 1, 0),      # Squeeze, ragged
    (1030, 770, 5, 6, 1, 2),     # RCT + Squeeze + weighted predictor
    (1024, 1024, 6, 6, 1, 1),
    (700, 530, 7, 6, 0, 3),      # reference-channel properties (17, 19)
    (513, 300, 8, 0, 1, 3),      # ... with Squeeze (channels of different shapes never reference each other)
]


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


@pytest.mark.parametrize("case", CASES)
def test_synthetic_modular_parity(ctx, case):
    import synth
    from tests import oracle_binding as ob
    w, h, seed, rct, sq, tk = case
    data = synth.encode_modular(w, h, seed, rct, sq, tk)
    src = synth.modular_source(w, h, seed)
    ref, ref_planes = ob.decode_modular_file(data, planes=True)
    assert np.array_equal(ref, src)  # the oracle itself is lossless on this input
    for lanes in (1, 4):
        (out,), (planes,) = gpu_decode(ctx, [data], lanes)
        assert np.array_equal(planes, ref_planes)
        assert np.array_equal(out, src)


@pytest.mark.parametrize("case", [(300, 260, 21, 1), (700, 530, 22, 2), (1030, 770, 23, 0)])
def test_palette_without_delta_entries_on_the_device(ctx, case):
    """a19: the global palette transform as a device look-up (transforms/palette.rs:165-199): explicit entries and both
    implicit colour cubes, index channel decoded by the group streams, palette meta channel by the host front-end."""
    import synth
    from tests import oracle_binding as ob
    w, h, seed, tk = case
    data = synth.encode_modular(w, h, seed, 0, 0, tk, palette=1)
    src = synth.modular_source(w, h, seed, palette=1)
    ref, ref_planes = ob.decode_modular_file(data, planes=True)
    assert np.array_equal(ref, src)
    (out,), (planes,) = gpu_decode(ctx, [data])
    assert np.array_equal(planes, ref_planes)
    assert np.array_equal(out, src)


@pytest.mark.parametrize("name", ["green_queen_modular_e3.jxl", "grayscale_public_university.jxl", "issue865_large_toc.jxl",
                                  "3x3_srgb_lossless.jxl", "lz77_flower.jxl", "tree_max_property_20.jxl"])
def test_real_modular_files(ctx, golden_dir, name):
    from tests import oracle_binding as ob
    data = open(os.path.join(golden_dir, "jxl", name), "rb").read()
    ref, ref_planes = ob.decode_modular_file(data, planes=True)
    (out,), (planes,) = gpu_decode(ctx, [data])
    assert np.array_equal(planes, ref_planes)
    assert np.array_equal(out, ref)


@pytest.mark.parametrize("name", ["delta_palette.jxl"])
def test_unsupported_modular_features_fail_loudly(ctx, golden_dir, name):
    """No CPU fallback: features outside the device scope are an error, not a silent host decode. (lz77_flower and
    tree_max_property_20 are single-group images: their channels are the "global" section 0, host front-end work.)"""
    import torch
    import jxl_rs_b200 as j
    data = open(os.path.join(golden_dir, "jxl", name), "rb").read()
    fr = j.ModularParsedFrame(data)
    out = torch.empty((fr.height, fr.width, 3), dtype=torch.uint8)
    b = j.ModularBatch(ctx)
    with pytest.raises(abi.JxgError) as e:
        b.add(fr, out.data_ptr(), fr.width * 3, False)
        b.run()
        b.wait()
    assert e.value.code == -2
    b.close()


def test_corrupt_modular_stream_reports_group(ctx):
    import synth
    import jxl_rs_b200 as j
    import torch
    data = bytearray(synth.encode_modular(600, 520, 9, 6, 0, 1))
    data[-2000] ^= 0x5A  # inside the last group's section
    fr = j.ModularParsedFrame(bytes(data))
    out = torch.empty((fr.height, fr.width, 3), dtype=torch.uint8).pin_memory()
    b = j.ModularBatch(ctx)
    b.add(fr, out.data_ptr(), fr.width * 3, False)
    b.run()
    with pytest.raises(abi.JxgError) as e:
        b.wait()
    assert e.value.code in (-7, -3)
    b.close()


def test_modular_batch_roundtrip_4k(ctx):
    """BASELINE config 5 geometry (reduced count): a batch of 4096x4096 lossless frames decodes to the source images."""
    import synth
    files = [synth.encode_modular(4096, 4096, 100 + i, 6, i % 2, 1) for i in range(2)]
    outs, _ = gpu_decode(ctx, [files[0]], 4)
    assert np.array_equal(outs[0], synth.modular_source(4096, 4096, 100))
    outs, _ = gpu_decode(ctx, [files[1]], 4)
    assert np.array_equal(outs[0], synth.modular_source(4096, 4096, 101))
