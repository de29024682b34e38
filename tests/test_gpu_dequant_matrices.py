"""Custom dequantisation matrices through the CUDA dequant + IDCT kernels: stage A of the GPU against f64 stage A built
from the encodings each frame was written with (tests/f64_quant.py), stages B and C on top (tests/gpu_stages.py).

Every table index 0-16 carries a custom table in frames whose varblocks read it, so that each kernel route reads one
from the frame's blob (F.dequant_off[qt] >= 0):
  - k_idct_small (is_small_reg_type): tables 0, 3, 4, 6 and 9;
  - the warp path of k_dequant_idct: the 32-row DCTs (tables 5, 7, 8) and IDENTITY, DCT2X2, AFV (tables 1, 2, 10);
  - the CTA path of k_dequant_idct: tables 11-16.
RAW tables with random entries sit at the square indices 0 and 11 and the non-square index 6. A mixed batch puts
frames with different custom tables for the same index, library tables and a shared custom table side by side."""
import pytest

from tests import f64_quant as fq
from tests.gpu_stages import check_frames

pytestmark = pytest.mark.gpu

# (width, height, seed) of profile-4 frames that place a varblock of every table index
ALL_TABLES = [(512, 512, 14), (768, 512, 12)]


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


def _frame(size, encs, epf=2, gab=1, x_qm_scale=3, b_qm_scale=2):
    """A profile-4 frame written with `encs`; asserts that every custom table is read by a varblock."""
    import jxl_rs_b200 as j
    import synth
    from jxl_rs_b200 import abi
    from tests import f64_pipeline as fp
    w, h, seed = size
    data = synth.encode_synthetic(w, h, seed, 1.0, epf, gab, 4, dequant=encs, x_qm_scale=x_qm_scale,
                                  b_qm_scale=b_qm_scale)
    if encs is not None:
        pf = j.ParsedFrame(data)
        fq.assert_custom_tables_used(fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0], encodings=encs), encs, str(size))
    return data


# (size, encodings seed, mode overrides, EPF, Gaborish, x_qm_scale, b_qm_scale)
CASES = [
    (ALL_TABLES[0], 1, {}, 2, 1, 3, 2),
    (ALL_TABLES[0], 2, {4: fq.MODE_RAW, 12: fq.MODE_RAW, 15: fq.MODE_RAW}, 1, 0, 0, 7),  # RAW on 16x16, 32x64, 256x256
    (ALL_TABLES[1], 3, {0: fq.MODE_DCT, 1: fq.MODE_DCT, 2: fq.MODE_DCT, 3: fq.MODE_DCT, 9: fq.MODE_DCT,
                        10: fq.MODE_DCT, 16: fq.MODE_RAW}, 3, 1, 7, 0),                  # DCT mode on the 8x8 tables
    (ALL_TABLES[0], 21, {5: fq.MODE_RAW}, 2, 1, 3, 2),                                    # RAW on 32x32
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0][0]}x{c[0][1]}-enc{c[1]}-xqm{c[5]}-bqm{c[6]}" for c in CASES])
def test_custom_tables_match_f64(ctx, case):
    size, es, modes, epf, gab, xq, bq = case
    encs = fq.profile4_encodings(es, modes)
    check_frames(ctx, [_frame(size, encs, epf, gab, xq, bq)], f"custom tables {case[:2]}", [encs])


def test_mixed_batch_matches_f64(ctx):
    """One batch: two frames with different custom tables at every index, a frame with library tables, and a frame
    sharing the first frame's custom tables. Each frame must meet its own reference, so a per-frame blob offset that
    points at another frame's table fails."""
    ea, eb = fq.profile4_encodings(11), fq.profile4_encodings(12)
    datas = [_frame(ALL_TABLES[0], ea), _frame(ALL_TABLES[0], eb), _frame(ALL_TABLES[0], None),
             _frame(ALL_TABLES[1], ea)]
    check_frames(ctx, datas, "mixed dequant batch", [ea, eb, None, ea])
