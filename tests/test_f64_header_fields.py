"""The oracle's VarDCT float path against float64 (tests/f64_pipeline.py) on frames whose header fields leave their
defaults: per-channel Gaborish weights, custom EPF sharpness LUTs, channel scales and sigma fields, every color_factor
encoding with negative and cancelling base correlations, CfL tile maps at and beyond the i8 ends, distinct opsin and
quant biases. Every frame is written by synth.encode_synthetic(header=...) and checked with f64_pipeline.Frame(header=),
so the f64 side takes each parameter from what the test wrote and the descriptor must hold the same values. Also: the
refusals of the header with a valid twin each, the token-level frames of test_vardct_ref.py through stages A-C, and
planted faults on the f64 side that frames with default headers would not catch. No GPU."""
import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import f64_header as fh
from tests import f64_pipeline as fp
from tests.test_f64_pipeline import _check_file, _stage_a_fails, _stage_b_fails

H = fh.f16_bits


def near(v):
    """The nearest f16 bit patterns of values."""
    return [int(x) for x in np.asarray(v, np.float16).view(np.uint16)]


def cfl_values(w, h, values):
    """CfL maps (ytox, ytob) of a w x h frame cycling through `values` (ytob in reverse order)."""
    n = ((h + 7) // 8 + 7) // 8 * (((w + 7) // 8 + 7) // 8)
    v = list(values)
    return [v[i % len(v)] for i in range(n)], [v[::-1][i % len(v)] for i in range(n)]


GAB = [H(0.09375), H(0.046875), H(-0.1875), H(0.125), H(0.140625), H(0.078125)]  # Y: T = 0.75, S = 2.25
SHARP = [H(0.5), H(0.0), H(-0.25), H(1.0), H(0.125), H(0.75), H(0.375), H(0.875)]  # non-monotone, 0, < 0
WEIGHT = [H(5.0), H(3.5), H(40.0), H(0.5), H(0.75)]                                  # channel scales rotated
SIGMA = [H(0.75), H(1.25), H(4.5), H(0.25)]                                          # quant_mul, pass0, pass2, border
OPSIN = {"matrix": near(fh.DEFAULTS["opsin_inverse_matrix"]),
         "biases": [H(-0.001953125), H(-0.0048828125), H(-0.00390625)],
         "quant_biases": [H(0.9375), H(0.875), H(0.96875), H(0.125)]}
CFL_EDGES = (-128, 127, 43, -43, 300, -1000, 0, 5, 128, -129)
SIGMA_DEFAULTS = near([0.9, 6.5, 2 / 3])  # pass0, pass2, border_sad_mul


def headers(w, h):
    """The header parameter sets, by name, for a w x h frame."""
    return {
        "gab": {"gab": GAB},
        "sharp": {"sharp": SHARP},
        "weight": {"weight": WEIGHT},
        "sigma": {"sigma": SIGMA},
        "factor256_cancel": {"color": {"factor": (1, 0), "base_x": H(-0.5), "base_b": H(4.0), "ytox_lf": -20,
                                       "ytob_lf": 17},
                             "cfl": cfl_values(w, h, (128, 127, 43, -43))},
        "factor8bit": {"color": {"factor": (2, 82), "base_x": H(-0.5), "base_b": H(-1.5), "ytox_lf": 127,
                                 "ytob_lf": -128}, "cfl": cfl_values(w, h, (42, -128, 7))},
        "factor16bit": {"color": {"factor": (3, 1000), "base_x": H(0.25), "base_b": H(0.5)},
                        "cfl": cfl_values(w, h, CFL_EDGES)},
        "factor84_cancel": {"color": {"factor": (0, 0), "base_x": H(-0.5), "base_b": H(1.0)},
                            "cfl": cfl_values(w, h, (43, 42, -128, 127))},
        "cfl_edges": {"cfl": cfl_values(w, h, CFL_EDGES)},
        "opsin": {"opsin": OPSIN},
        # every LUT entry puts the blocks of raw_quant 5 (global_scale 4587, distance 1) within one f32 ulp of
        # MIN_SIGMA: f32 passes them through and float64 does not (keep), or the other way round (filter)
        "sigma_edge_keep": {"sharp": [0x3230] * 8, "sigma": [H(0.54296875)] + SIGMA_DEFAULTS},
        "sigma_edge_filter": {"sharp": [0x3180] * 8, "sigma": [H(0.61083984375)] + SIGMA_DEFAULTS},
        "all": {"gab": GAB, "sharp": SHARP, "weight": WEIGHT, "sigma": SIGMA, "opsin": OPSIN,
                "color": {"factor": (2, 40), "base_x": H(-0.25), "base_b": H(1.25), "ytox_lf": 5, "ytob_lf": -9},
                "cfl": cfl_values(w, h, CFL_EDGES)},
    }


# (width, height, seed, distance, epf_iters, gab, profile, entropy, colour) per header set; "all" at every EPF x Gaborish
CASES = ([(name, (300, 280, 30 + i, 1.0, 2, 1, 1, 0, 0)) for i, name in enumerate(headers(1, 1))]
         + [(name, (129, 97, 50 + i, 1.0, 3, 1, 1, 0, 0)) for i, name in enumerate(("gab", "sharp", "weight", "sigma"))]
         + [(name, (200, 264, 60 + i, 0.7, 1, 0, 3, 0, 0)) for i, name in enumerate(("factor8bit", "cfl_edges"))]
         + [("all", (96, 80, 70 + 2 * epf + gab, 1.0, epf, gab, 1, 0, 0)) for epf in range(4) for gab in (0, 1)]
         + [("all", (520, 512, 80, 1.0, 2, 1, 3, 0, 0))]
         + [(name, (300, 280, 202, 1.0, 2, 1, 1, 0, 0)) for name in ("sigma_edge_keep", "sigma_edge_filter")])


def written(case, name):
    import synth
    w, h, seed, dist, epf, gab, profile, entropy, colour = case
    header = headers(w, h)[name]
    return synth.encode_synthetic(w, h, seed, dist, epf, gab, profile, entropy=entropy, colour=colour,
                                  header=header), header


def _frame(data, header):
    import jxl_rs_b200 as j
    pf = j.ParsedFrame(data)  # owns the descriptor's arrays while Frame copies them
    return fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0], header=header)


@pytest.mark.parametrize("name,case", CASES, ids=[f"{n}-{c[0]}x{c[1]}-epf{c[4]}-gab{c[5]}" for n, c in CASES])
def test_header_frames_match_f64(name, case):
    """Stages A, B and C of the oracle (every output format) on a frame written with the header set; the f64 side
    takes the parameters from the header (Frame(header=) asserts that the descriptor holds them)."""
    data, header = written(case, name)
    fr = _frame(data, header)
    if "opsin" in header:  # sRGB output: the descriptor's output matrix is the one written
        assert np.array_equal(fr.opsin_inverse_matrix, fr.written_opsin_matrix)
    print(name, case, _check_file(data, name, header))


def test_header_frames_reach_their_edges():
    """The header sets put what they are for into the frames: CfL values clamped at both ends, blocks passed through
    by a LUT entry <= 0, an x_cc cancelled to near 0, per-channel Gaborish weights with a negative one."""
    data, header = written((300, 280, 30, 1.0, 2, 1, 1, 0, 0), "all")
    fr = _frame(data, header)
    assert fr.ytox.min() == -128 and fr.ytox.max() == 127 and fr.ytob.min() == -128 and fr.ytob.max() == 127
    keep = fp.pass_through_f32(fr.global_scale, fr.raw_quant, fr.epf_map, fr.epf_quant_mul, fr.epf_sharp_lut)
    assert keep.any() and (~keep).any() and (fr.epf_sharp_lut[fr.epf_map][keep] <= 0).any()
    assert (fr.gab_w1 < 0).any() and len(set(fr.gab_w1)) == 3 and len(set(fr.gab_w2)) == 3
    data, header = written((300, 280, 30, 1.0, 2, 1, 1, 0, 0), "factor84_cancel")
    fr = _frame(data, header)
    assert (np.abs(fr.base_x + fr.ytox / fr.color_factor) < 0.02).any()


def threshold_blocks(fr):
    """Blocks whose f32 1 / sigma lies within one f32 ulp of MIN_SIGMA, and blocks where the f32 pass-through decision
    (f64_pipeline.pass_through_f32) differs from the float64 one. Returns (near, differ, keep)."""
    keep = fp.pass_through_f32(fr.global_scale, fr.raw_quant, fr.epf_map, fr.epf_quant_mul, fr.epf_sharp_lut)
    f = np.float32
    quant_scale = f(1.0) / (f(65536.0) / f(fr.global_scale))
    sq = f(fr.epf_quant_mul) / (quant_scale * fr.raw_quant.astype(f) * f(fp.INV_SIGMA_NUM))
    inv = f(1.0) / np.minimum(sq * fr.epf_sharp_lut.astype(f)[fr.epf_map], f(-1e-4))
    ulps = np.abs(inv.view(np.int32).astype(np.int64) - int(np.array(f(fp.MIN_SIGMA)).view(np.int32)))
    s64 = fp.sigma_image_f64(fr.global_scale, fr.raw_quant, fr.epf_map, fr.epf_quant_mul, fr.epf_sharp_lut)
    return ulps <= 1, keep != (s64 < fp.MIN_SIGMA), keep


@pytest.mark.parametrize("name", ["sigma_edge_keep", "sigma_edge_filter"])
def test_blocks_on_the_epf_threshold(name):
    """Blocks within one f32 ulp of MIN_SIGMA, with blocks passed through and blocks filtered in the same frame, and
    blocks where the f32 and float64 decisions part (f32 keeps them in one set, filters them in the other). Stage B
    holds with the decision taken on the f32 sigma, and fails when it is taken on the float64 sigma (the planted fault;
    default frames would not catch it, since none of their blocks lies within f32 rounding of the threshold)."""
    data, header = written((300, 280, 202, 1.0, 2, 1, 1, 0, 0), name)
    fr = _frame(data, header)
    on, differ, keep = threshold_blocks(fr)
    assert on.any() and differ.any() and keep.any() and (~keep).any()
    assert (keep[differ] == (name == "sigma_edge_keep")).all()
    _check_file(data, name, header)
    import unittest.mock as um  # the planted fault: decide on the float64 sigma
    with um.patch.object(fp, "pass_through_f32", lambda gs, rq, sh, qm, lut: fp.sigma_image_f64(gs, rq, sh, qm, lut)
                         < fp.MIN_SIGMA):
        _stage_b_fails(data, fr)


def test_round_trip_with_custom_header():
    """The writer quantises with the colour correlation and opsin fields it writes: the decode reproduces the source
    (PSNR > 30 dB, as test_cpu_paths.test_synthetic_writer_round_trip for default headers). Gaborish and EPF
    fields are not inverted by the writer, so this frame keeps them at their defaults."""
    import synth
    from tests import oracle_binding as ob
    from tests.test_cpu_paths import _srgb_exact
    w, h = 300, 200
    hd = {k: v for k, v in headers(w, h)["all"].items() if k in ("color", "opsin", "cfl")}
    data = synth.encode_synthetic(w, h, 7, 0.5, 2, 1, 1, header=hd)
    out, _ = ob.decode_file(data, abi.FORMAT_RGB_F32, threads=4)
    src = _srgb_exact(synth.modular_source(w, h, 7) / 255.0)
    mse = float(np.mean((out.astype(np.float64) - src) ** 2))
    assert 10 * np.log10(1.0 / mse) > 30.0, f"PSNR {10 * np.log10(1.0 / mse):.1f} dB"


# ---------------------------------------------------------------------------------------------------------------------
# The descriptor against the written values, and the refusals with their valid twins
# ---------------------------------------------------------------------------------------------------------------------
NAN, INF = 0x7E00, 0x7C00
ABOVE_4 = 0x4401  # the next f16 above 4.0


def _refusals():
    """(name, valid header, refused header): each twin differs in one field."""
    out = [("base_x_above_4", {"color": {"base_x": H(4.0)}}, {"color": {"base_x": ABOVE_4}}),
           ("base_b_above_4", {"color": {"base_b": H(4.0)}}, {"color": {"base_b": ABOVE_4}}),
           ("base_x_nan", {"color": {"base_x": H(-4.0)}}, {"color": {"base_x": NAN}}),
           ("base_b_inf", {"color": {"base_b": H(-100.0)}}, {"color": {"base_b": 0xFC00}})]
    for key, good in (("gab", GAB), ("sharp", SHARP), ("weight", WEIGHT), ("sigma", SIGMA)):
        for i, bad in ((0, NAN), (len(good) - 1, INF)):
            out.append((f"{key}{i}_{'nan' if bad == NAN else 'inf'}", {key: good}, {key: good[:i] + [bad] + good[i + 1:]}))
    for part in ("matrix", "biases", "quant_biases"):
        bad = dict(OPSIN)
        bad[part] = [NAN] + OPSIN[part][1:]
        out.append((f"opsin_{part}_nan", {"opsin": OPSIN}, {"opsin": bad}))
    return out


REFUSALS = _refusals()


@pytest.mark.parametrize("name,good,bad", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusal_with_twin(name, good, bad):
    """The valid twin parses and its descriptor holds the written values; the refused header is refused by the front
    end, by the oracle and by the f64 restatement. Negative bases are accepted, as in the reference."""
    import jxl_rs_b200 as j
    import synth
    from tests import oracle_binding as ob
    gd = synth.encode_synthetic(64, 64, 3, 1.0, 2, 1, 1, header=good)
    fr = _frame(gd, good)
    ob.decode_file(gd, abi.FORMAT_RGB_U8)
    assert fr.width == 64
    bd = synth.encode_synthetic(64, 64, 3, 1.0, 2, 1, 1, header=bad)
    with pytest.raises(fh.Refused):
        fh.decode(bad)
    with pytest.raises(Exception):
        j.ParsedFrame(bd)
    with pytest.raises(Exception):
        ob.decode_file(bd, abi.FORMAT_RGB_U8)


def test_skipped_groups_keep_defaults():
    """With Gaborish off and EPF 0 the reader skips the custom groups: a header dict that holds them writes nothing,
    and the descriptor keeps the defaults (the f64 side, which takes the values from decode(), agrees)."""
    import synth
    hd = {"gab": GAB, "sharp": SHARP, "weight": WEIGHT, "sigma": SIGMA}
    fr = _frame(synth.encode_synthetic(64, 64, 3, 1.0, 0, 0, 1, header=hd), hd)
    assert fr.epf_iters == 0 and fr.gab == 0
    assert np.array_equal(fr.gab_w1, fh.DEFAULTS["gab_w1"]) and np.array_equal(fr.epf_sharp_lut, fh.DEFAULTS["epf_sharp_lut"])


def test_default_frame_without_header_and_custom_frame_refused():
    """Frame without `header` accepts a default frame and refuses one with custom fields, naming them."""
    import jxl_rs_b200 as j
    import synth
    pf = j.ParsedFrame(synth.encode_synthetic(64, 64, 3, 1.0, 2, 1, 1))
    fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0])
    hd = headers(64, 64)["all"]
    pf = j.ParsedFrame(synth.encode_synthetic(64, 64, 3, 1.0, 2, 1, 1, header=hd))
    with pytest.raises(ValueError, match="non-default header fields"):
        fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0])
    fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0], header=hd)


def test_opsin_inverse_fixture_literals():
    """opsin_inverse.jxl's custom opsin fields, held as f16 literals, are what the front end parses."""
    import jxl_rs_b200 as j
    data = open(fp.os.path.join(fp.ROOT, "tests/golden/jxl/opsin_inverse.jxl"), "rb").read()
    pf = j.ParsedFrame(data)
    fr = fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0], header=fh.OPSIN_INVERSE_FIXTURE)
    assert np.array_equal(fr.opsin_inverse_matrix, fr.written_opsin_matrix)
    assert len(set(fr.opsin_biases)) == 3


# ---------------------------------------------------------------------------------------------------------------------
# Token-level frames (test_vardct_ref.CASES) through stages A-C
# ---------------------------------------------------------------------------------------------------------------------
def _token_cases():
    from tests import test_vardct_ref as T
    return T.CASES


# The token frames run again with non-default colour correlation and CfL maps: factor 256 (selector 1), bases that
# cancel map / factor (-0.25 + 64 / 256 = 0; 65 gives 0.004) and negative, LF factors, maps at and beyond the i8 ends
TOKEN_CFL_CASES = ["passes11", "passes2_wrap", "entry_edges", "shapes_large"]


def token_header(w, h):
    return {"color": {"factor": (1, 0), "base_x": H(-0.25), "base_b": H(-0.5), "ytox_lf": 64, "ytob_lf": -100},
            "cfl": cfl_values(w, h, (64, 65, -128, 127, 300, -1000, 128, 0))}


def token_frame(name, cfl=False):
    """(model frame, file bytes, header) of a token-level frame, with token_header when cfl is set; the coefficients
    are the model's either way (the header does not touch the AC streams)."""
    import synth
    from tests import test_vardct_ref as T
    f, data = T.model(name)
    if not cfl:
        return f, data, None
    header = token_header(f.spec["width"], f.spec["height"])
    return f, synth.encode_vardct_tokens(dict(f.spec, header={"color": header["color"]}, cfl=header["cfl"])), header


TOKEN_CASES = [(n, False) for n in _token_cases()] + [(n, True) for n in TOKEN_CFL_CASES]


@pytest.mark.parametrize("name,cfl", TOKEN_CASES, ids=[n + ("-cfl" if c else "") for n, c in TOKEN_CASES])
def test_token_frames_match_f64(name, cfl):
    """Each token-level frame on the oracle: coefficients equal to the model's, then stages A, B and C in every output
    format. These frames reach the coefficient-entry edges (entry_edges: +-2^25 for 8x8, +-2^15 for DCT256), 11 shifted
    passes, every order up to 256x256 and ragged frames; four of them again with token_header's colour correlation."""
    from tests import oracle_binding as ob
    f, data, header = token_frame(name, cfl)
    fr = _frame(data, header)
    if cfl:
        assert fr.ytox.min() == -128 and fr.ytox.max() == 127 and (np.abs(fr.base_x + fr.ytox / fr.color_factor) < 0.01).any()
    out, taps = ob.decode_file(data, abi.FORMAT_RGB_F32, taps=True)
    assert np.array_equal(taps["coeffs"], f.coeffs), name
    a, ma = fp.stage_a(fr, taps["coeffs"])
    ratios = [fp.check("A", taps["xyb_idct"], a, ma, name)]
    b, mb = fp.stage_b(fr, taps["xyb_idct"].astype(np.float64))
    ratios.append(fp.check("B", taps["xyb_filtered"], b, mb, name))
    ratios.append(check_c_in_f32_range(data, header, taps["xyb_filtered"], out, name))
    print(name, cfl, "largest err/(2^-24 M) per stage (A, B, C):", ratios)


def check_c_in_f32_range(data, header, xyb, out_f32, what):
    """Stage C of the oracle in every output format where an f32 implementation can compute it
    (f64_pipeline.srgb_f32_overflow): the entry-edge and shifted multi-pass frames reach XYB planes of 4e6-8e6, and the
    sRGB curve overflows f32 on their largest linear values. Those samples are left out of the f32 check and may take
    any code in the integer and half stores; they must be under 1% of the frame. Every other sample is held to the
    bound. Returns the largest err / (2^-24 M) of the f32 output."""
    import jxl_rs_b200 as j
    from tests import oracle_binding as ob
    from tests.test_f64_pipeline import FORMATS
    xyb = np.asarray(xyb, np.float64)
    pf = j.ParsedFrame(data)
    outs = {abi.FORMAT_RGB_F32: out_f32}
    ratio = 0.0
    for fmt in FORMATS:
        fr = fp.Frame(pf.desc(fmt)[0], header=header)
        got = outs[fmt] if fmt in outs else ob.decode_file(data, fmt)[0]
        c, mc = fp.stage_c(fr, xyb)
        over = fp.srgb_f32_overflow(fr, xyb)
        assert over.sum() <= over.size // 100, f"{what}: {int(over.sum())} samples beyond the f32 range of the curve"
        if fmt == abi.FORMAT_RGB_F32:
            ratio = fp.check("C", np.asarray(got)[~over], c[~over], mc[~over], what)
        else:  # any code at those samples, NaN included (an f16 store of inf / inf): replaced by 0 before the check
            got = np.array(got, copy=True)
            got[..., :3][over] = 0
            fp.check_output(fmt, got, c, np.where(over, np.inf, mc), fr.output_tf, 1, f"{what} format {fmt}")
    return ratio


# ---------------------------------------------------------------------------------------------------------------------
# Planted faults on the f64 side: each must fail its bound on a frame written with the field non-default
# ---------------------------------------------------------------------------------------------------------------------
def _fault_frame(name, case=(300, 280, 30, 1.0, 2, 1, 1, 0, 0)):
    data, header = written(case, name)
    return data, _frame(data, header)


def test_fault_gaborish_weights_of_channel_0_for_all():
    """Channel 0's Gaborish weights used for all three channels. Default frames: not caught (the weights are equal in
    X, Y and B)."""
    data, fr = _fault_frame("gab")
    fr.gab_w1, fr.gab_w2 = np.full(3, fr.gab_w1[0]), np.full(3, fr.gab_w2[0])
    _stage_b_fails(data, fr)


def test_fault_sharp_lut_linear():
    """The sharpness LUT replaced by i / 7. Default frames: not caught (their LUT is i / 7)."""
    data, fr = _fault_frame("sharp")
    fr.epf_sharp_lut = np.arange(8) / 7.0
    _stage_b_fails(data, fr)


def test_fault_channel_scales_rotated():
    """The EPF channel scales rotated by one channel. Default frames: caught (40, 5, 3.5 are distinct); here the
    written scales are themselves rotated, so the fault restores the default order."""
    data, fr = _fault_frame("weight")
    fr.epf_channel_scale = np.roll(fr.epf_channel_scale, 1)
    _stage_b_fails(data, fr)


def test_fault_border_sad_mul_ignored():
    """epf_border_sad_mul taken as 1. Default frames: caught (2/3); kept so that a custom value is followed."""
    data, fr = _fault_frame("sigma")
    fr.epf_border_sad_mul = 1.0
    _stage_b_fails(data, fr)


def test_fault_pass0_pass2_sigma_scales_swapped():
    """The pass 0 and pass 2 sigma scales swapped, on an EPF 3 frame. Default frames: caught (0.9 and 6.5)."""
    data, fr = _fault_frame("sigma", (129, 97, 53, 1.0, 3, 1, 1, 0, 0))
    fr.epf_pass0_sigma_scale, fr.epf_pass2_sigma_scale = fr.epf_pass2_sigma_scale, fr.epf_pass0_sigma_scale
    _stage_b_fails(data, fr)


def test_fault_quant_mul_fixed():
    """epf_quant_mul fixed at 0.46. Default frames: not caught (0.46 is the default)."""
    data, fr = _fault_frame("sigma")
    fr.epf_quant_mul = 0.46
    _stage_b_fails(data, fr)


def test_fault_color_factor_fixed_at_84():
    """color_factor fixed at 84. Default frames: not caught (84 is the default)."""
    data, fr = _fault_frame("factor256_cancel")
    assert fr.color_factor == 256
    fr.color_factor = 84
    _stage_a_fails(data, fr)


def test_fault_bases_swapped():
    """base_correlation_x and base_correlation_b swapped. Default frames: caught (0 and 1); here the bases are -0.5
    and -1.5."""
    data, fr = _fault_frame("factor8bit")
    fr.base_x, fr.base_b = fr.base_b, fr.base_x
    _stage_a_fails(data, fr)


def test_fault_cfl_map_wrapped_as_i8():
    """The CfL map values wrapped to i8 instead of clamped (300 -> 44, 128 -> -128). Default frames: not caught (their
    values lie in [-8, 8])."""
    data, fr = _fault_frame("cfl_edges")
    w, h = 300, 280
    raw = [np.asarray(m, np.int64).reshape(fr.ytox.shape) for m in headers(w, h)["cfl_edges"]["cfl"]]
    fr.ytox, fr.ytob = ((m.astype(np.int8)).astype(np.int32) for m in raw)
    _stage_a_fails(data, fr)


def test_fault_opsin_bias_0_for_all():
    """opsin_biases[0] used for all channels. Default frames: not caught (the biases are equal)."""
    from tests import oracle_binding as ob
    data, fr = _fault_frame("opsin")
    out, taps = ob.decode_file(data, abi.FORMAT_RGB_F32, taps=True)
    xyb = taps["xyb_filtered"].astype(np.float64)
    c, mc = fp.stage_c(fr, xyb)
    fp.check("C", out, c, mc)
    fr.opsin_biases = np.full(3, fr.opsin_biases[0])
    c, mc = fp.stage_c(fr, xyb)
    with pytest.raises(AssertionError):
        fp.check("C", out, c, mc)
