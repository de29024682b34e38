"""The CUDA float path against float64 (tests/gpu_stages.check_frames) on frames whose header fields leave their defaults
(the parameter sets of test_f64_header_fields.py), on both paths of the fused filter kernel:
  - Gaborish + EPF 2 at sizes with aligned interior tiles, where filter_tile_v4 runs (asserted per output format with
    test_gpu_output_stage.vector_tiles), its scalar edges, and EPF 0 / 1 / 3 and Gaborish off on filter_tile;
  - non-default CfL (maps at and beyond the i8 ends, every color_factor encoding, cancelling bases) on every transform
    route: k_idct_small, the warp and CTA paths of k_dequant_idct (profile 3), with varblocks that span several CfL
    tiles and a ragged frame whose last tile column is partial;
  - blocks within one f32 ulp of the EPF pass-through threshold, on both filter paths;
  - one batch of frames sharing a (Gaborish, EPF) configuration with different parameters, plus a default frame;
  - the token-level frames of test_vardct_ref.py, with coefficients equal to the model's, four of them again with
    non-default colour correlation and CfL maps."""
import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import test_f64_header_fields as HF
from tests.gpu_stages import check_frames
from tests.test_gpu_output_stage import vector_tiles

pytestmark = pytest.mark.gpu

VECTOR_FORMATS = (abi.FORMAT_XYB_F32_PLANAR, abi.FORMAT_RGB_F32, abi.FORMAT_RGB_U8)  # the formats check_frames runs
BPP = {abi.FORMAT_XYB_F32_PLANAR: 4, abi.FORMAT_RGB_F32: 12, abi.FORMAT_RGB_U8: 3}


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


def _vector_path_runs(case):
    w, h, epf, gab = case[0], case[1], case[4], case[5]
    return all(vector_tiles(w, h, gab, epf, f, w * BPP[f]) > 0 for f in VECTOR_FORMATS)


# (header set, (width, height, seed, distance, epf_iters, gab, profile, entropy, colour))
VECTOR = [(name, (520, 512, 100 + i, 1.0, 2, 1, 1, 0, 0)) for i, name in enumerate(HF.headers(1, 1))]
SCALAR = ([(name, (129, 97, 120 + i, 1.0, 2, 1, 1, 0, 0)) for i, name in enumerate(("gab", "sigma", "weight", "sharp"))]
          + [("all", (96, 80, 130 + 2 * epf + gab, 1.0, epf, gab, 1, 0, 0)) for epf in range(4) for gab in (0, 1)
             if (epf, gab) != (2, 1)])
# profile 3: DCT128 / 256 families on the CTA path, 32-row DCTs on the warp path, small DCTs in k_idct_small; the
# large varblocks span several 64x64 CfL tiles; 200 wide: the last tile column holds 8 of 64 pixels
CFL = [(name, (w, h, 140 + i, 0.7, 2, 1, 3, 0, 0)) for i, (name, (w, h)) in enumerate(
    [("cfl_edges", (520, 512)), ("factor256_cancel", (520, 512)), ("factor8bit", (200, 264)),
     ("factor16bit", (200, 264)), ("factor84_cancel", (776, 520)), ("all", (200, 264))])]


def _ids(cases):
    return [f"{n}-{c[0]}x{c[1]}-epf{c[4]}-gab{c[5]}-p{c[6]}" for n, c in cases]


def _check(ctx, cases, what):
    import jxl_rs_b200 as j
    from tests import f64_pipeline as fp
    datas, headers = zip(*(HF.written(c, n) for n, c in cases))
    for data, header in zip(datas, headers):
        if "opsin" in header:  # sRGB output: stage C's matrix (the descriptor's output matrix) is the one written
            pf = j.ParsedFrame(data)
            fr = fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0], header=header)
            assert np.array_equal(fr.opsin_inverse_matrix, fr.written_opsin_matrix)
    return check_frames(ctx, list(datas), what, headers=list(headers))


@pytest.mark.parametrize("name,case", VECTOR, ids=_ids(VECTOR))
def test_vector_path_header_fields(ctx, name, case):
    assert _vector_path_runs(case)
    _check(ctx, [(name, case)], f"vector {name}")


@pytest.mark.parametrize("name,case", SCALAR, ids=_ids(SCALAR))
def test_scalar_path_header_fields(ctx, name, case):
    assert not _vector_path_runs(case)
    _check(ctx, [(name, case)], f"scalar {name}")


@pytest.mark.parametrize("name,case", CFL, ids=_ids(CFL))
def test_cfl_on_every_transform_route(ctx, name, case):
    import jxl_rs_b200 as j
    from tests import f64_pipeline as fp
    data, header = HF.written(case, name)
    pf = j.ParsedFrame(data)
    fr = fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0], header=header)
    types = set((fr.transform_map[fr.transform_map >= 128] & 127).tolist())
    # CTA, warp and small routes; 21-26 (128 and 256 pixels on a side) span several 64x64 CfL tiles
    assert types & set(range(21, 27)) and types & {5, 8, 9, 10, 11} and 0 in types, types
    if case[0] % 64:
        assert (fr.xb % 8) != 0  # the last CfL tile column is partial
    _check(ctx, [(name, case)], f"cfl {name}")


# frames with blocks on the EPF threshold (test_f64_header_fields.threshold_blocks), on the vector and the scalar path
THRESHOLD = [("sigma_edge_keep", (520, 512, 200, 1.0, 2, 1, 1, 0, 0)),
             ("sigma_edge_filter", (520, 512, 200, 1.0, 2, 1, 1, 0, 0)),
             ("sigma_edge_keep", (129, 97, 212, 1.0, 2, 1, 1, 0, 0)),
             ("sigma_edge_filter", (129, 97, 209, 1.0, 2, 1, 1, 0, 0))]


@pytest.mark.parametrize("name,case", THRESHOLD, ids=_ids(THRESHOLD))
def test_blocks_on_the_epf_threshold(ctx, name, case):
    data, header = HF.written(case, name)
    on, differ, keep = HF.threshold_blocks(HF._frame(data, header))
    assert on.any() and differ.any() and keep.any() and (~keep).any()
    assert _vector_path_runs(case) == (case[0] == 520)
    _check(ctx, [(name, case)], f"threshold {name}")


def test_batch_of_distinct_parameters_per_frame(ctx):
    """Frames sharing Gaborish + EPF 2 (one filter launch range) with different header fields, and a default frame:
    each CTA must read its own frame's parameters, not the first frame's."""
    cases = [(n, (520, 512, 160 + i, 1.0, 2, 1, 1, 0, 0)) for i, n in enumerate(("gab", "sharp", "all", "opsin"))]
    datas, headers = zip(*(HF.written(c, n) for n, c in cases))
    import synth
    datas = list(datas) + [synth.encode_synthetic(520, 512, 170, 1.0, 2, 1, 1)]
    check_frames(ctx, datas, "distinct parameters batch", headers=list(headers) + [None])


@pytest.mark.parametrize("name,cfl", HF.TOKEN_CASES, ids=[n + ("-cfl" if c else "") for n, c in HF.TOKEN_CASES])
def test_token_frames_through_stages(ctx, name, cfl):
    """Each token-level frame through stages A-C on the GPU, four of them again with test_f64_header_fields.token_header;
    the oracle's coefficients (which check_frames holds the GPU's to) equal the model's."""
    from tests import test_vardct_ref as T
    f, data, header = HF.token_frame(name, cfl)
    assert np.array_equal(T.oracle_coeffs(data), f.coeffs)
    check_frames(ctx, [data], f"tokens {name}{' cfl' if cfl else ''}", headers=[header])
