"""The CUDA VarDCT float path against the float64 restatement in tests/f64_pipeline.py, one stage at a time, each stage fed
the GPU's own input to it (tests/gpu_stages.py: A after dequant + IDCT, B the fused filter kernel, C the output stage).
Covers all eight (Gaborish, EPF 0-3) pairs, one-pixel edge tiles of the 64x32 filter tile,
transform profiles 0-3, prefix-coded streams, sRGB / linear / grey / PQ / BT.709 outputs, the fixtures with IDENTITY /
DCT2X2 / AFV varblocks and one batch mixing filter configurations."""
import os

import pytest

from tests.gpu_stages import check_frames as _check_frames

pytestmark = pytest.mark.gpu

# (width, height, seed, distance, epf_iters, gab, profile, entropy, colour)
SYNTHETIC = [
    (1, 1, 1, 1.0, 1, 1, 0, 0, 0),
    (3, 3, 2, 1.0, 0, 1, 1, 0, 0),
    (8, 8, 3, 1.0, 2, 0, 0, 0, 0),
    (9, 17, 4, 1.0, 3, 1, 1, 0, 0),
    (63, 65, 5, 1.0, 0, 0, 1, 0, 0),       # Gaborish off, EPF 0
    (263, 131, 6, 1.5, 2, 0, 2, 1, 0),     # Gaborish off, EPF 2; prefix-coded
    (129, 97, 7, 1.0, 1, 0, 1, 0, 0),      # 64k+1 x 32k+1: one-pixel edge tiles of the fused 64x32 filter tile
    (200, 264, 8, 0.7, 3, 0, 3, 0, 1),     # Gaborish off, EPF 3; 128 / 256 families; linear output
    (193, 129, 9, 1.0, 2, 1, 1, 0, 6),     # grey output
    (520, 512, 10, 1.0, 1, 1, 3, 0, 0),    # vector path inside, scalar path on the ragged edges
    (777, 513, 11, 0.5, 0, 1, 2, 0, 0),
    (600, 520, 12, 1.0, 2, 0, 1, 0, 0),    # Gaborish off, EPF 2, several groups
    (160, 96, 13, 1.0, 2, 1, 1, 0, 3),     # P3 + PQ output
    (160, 96, 14, 1.0, 1, 0, 1, 0, 5),     # custom primaries, DCI white, BT.709 output
]
# The fixtures with IDENTITY, DCT2X2 and AFV varblocks. progressive_ac (3.4 MP) also has them but is over the ~2 MP of
# f64 work per case; it is checked against the f64 stages on the oracle (test_f64_pipeline.py), and the GPU against the
# oracle in test_gpu_parity.py.
FIXTURES = ["zoltan_tasi_unsplash", "opsin_inverse", "dice"]


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


def _synthetic(case):
    import synth
    w, h, seed, dist, epf, gab, profile, entropy, colour = case
    return synth.encode_synthetic(w, h, seed, dist, epf, gab, profile, entropy=entropy, colour=colour)


@pytest.mark.parametrize("case", SYNTHETIC, ids=[f"{c[0]}x{c[1]}-epf{c[4]}-gab{c[5]}-p{c[6]}-e{c[7]}-c{c[8]}" for c in SYNTHETIC])
def test_synthetic_stages_match_f64(ctx, case):
    _check_frames(ctx, [_synthetic(case)], str(case))


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_stages_match_f64(ctx, name, golden_dir):
    _check_frames(ctx, [open(os.path.join(golden_dir, "jxl", name + ".jxl"), "rb").read()], name)


def test_mixed_filter_batch_matches_f64(ctx):
    """One batch of frames with different (Gaborish, EPF) pairs: the filter kernel runs once per configuration and CTAs of
    other configurations exit at once; every frame must still meet its own reference."""
    cases = [(96, 80, 20 + k, 1.0, epf, gab, 1, 0, 0) for k, (gab, epf) in enumerate([(0, 0), (1, 2), (0, 2), (1, 0), (0, 3), (1, 1)])]
    _check_frames(ctx, [_synthetic(c) for c in cases], "mixed batch")
