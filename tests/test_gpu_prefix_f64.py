"""The prefix decode on the GPU against float64, stage by stage, each stage fed the GPU's own input (gpu_stages.check_frames
with prefix handles; tests/f64_prefix.py):

  A  debug stop 2 against f64_prefix.stage_a: decoded groups from their coefficients, zero-pass groups the float64
     Upsample8x of the LF image (for token-level frames the float64 LF image of their LF integers)
  B  XYB_F32_PLANAR against stage B of the GPU's stage-A planes: the filters across the seams between upsampled and
     decoded groups, in both directions (permuted files put zero-pass groups left of and above decoded ones)
  C  RGB_F32 / RGB_U8 against stage C, the six formats and the eight orientations, and regions against the crop

on the files and cuts of test_prefix_f64.py: the end of HfGlobal, half way through the HF sections, permuted TOCs,
multi-pass token frames with 0, 1 and 2 passes per group, an arrived section past its group's pass count, and the edge
sizes of test_gpu_prefix. progressive_ac.jxl is over the f64 stages' budget (test_gpu_f64_stages.py) and stays with
test_gpu_prefix.py."""
import numpy as np
import pytest

import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from tests import f64_pipeline as fp
from tests import f64_prefix as fpx
from tests import gpu_stages as gs
from tests import prefix_ref as pr
from tests import test_prefix_f64 as P
from tests.test_gpu_prefix import decode, mid_cut

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = j.JxgContext(0)
    yield c
    c.close()


def _cut(data, kind):
    """start: the end of HfGlobal; mid: the end of the first half of the groups' pass-0 sections."""
    if kind == "start":
        return pr.prefix_start(data)
    off, ln = pr.hf_sections(data)
    g = max(0, off.shape[1] // 2 - 1)
    return int(off[0, g] + ln[0, g])


# (name, width, height, seed, keywords): the edge sizes of test_gpu_prefix / test_gpu_f64_stages
CUSTOM_W8 = np.random.default_rng(3).uniform(-0.05, 0.3, 210).astype(np.float16).view(np.uint16)
SYNTH = [("1100x700", 1100, 700, 401, {}),
         ("200x600-one-group-column", 200, 600, 402, {}),
         ("264x264-one-lf-sample-edge", 264, 264, 403, {}),
         ("513x289-one-pixel-tiles", 513, 289, 404, {}),
         ("520x512-vector-path", 520, 512, 405, {}),
         ("600x520-weights8", 600, 520, 406, {"header": {"weights8": CUSTOM_W8.tolist()}})]


@pytest.mark.parametrize("cut", ["start", "mid"])
@pytest.mark.parametrize("name,w,h,seed,kw", SYNTH, ids=[s[0] for s in SYNTH])
def test_synthetic_prefix_stages(ctx, name, w, h, seed, kw, cut):
    data = synth.encode_synthetic(w, h, seed, **kw)
    c = _cut(data, cut)
    k = j.PrefixParsedFrame(data[:c]).passes
    assert not k.any() if cut == "start" else (k.any() and not k.all())
    w8 = pr.f16_bits_to_float(CUSTOM_W8) if "header" in kw else None
    gs.check_frames(ctx, [data], f"{name} {cut}", headers=[kw.get("header")], cuts=[c], weights8=[w8])


def test_zero_pass_groups_left_of_and_above_decoded_ones(ctx):
    """The groups stored in reverse: zero-pass groups meet decoded ones on their right and bottom edges, and regions
    whose cones hold both kinds of seam."""
    data, cut = P.seam_case()
    regions = [(236, 300, 40, 40), (100, 492, 60, 40), (200, 450, 120, 120), (520, 500, 300, 30)]
    gs.check_frames(ctx, [data], "reverse-stored seam", cuts=[cut], regions=[regions])


def test_decoded_groups_above_zero_pass_ones(ctx):
    """The writer's order cut half way: decoded groups above and left of zero-pass ones, with regions over the seams."""
    data = synth.encode_synthetic(1100, 700, 301)
    cut = mid_cut(data)
    k = j.PrefixParsedFrame(data[:cut]).passes.reshape(-1, 5)
    assert k[0].all() and not k[-1].any()
    regions = [(0, 0, 1100, 700), (240, 236, 300, 40), (700, 480, 60, 60)]
    gs.check_frames(ctx, [data], "writer-order seam", cuts=[cut], regions=[regions])


def _token(name):
    spec = P.spec_of(name)
    data = synth.encode_vardct_tokens(spec)
    return spec, data


def _lf_image(spec, data):
    d = j.ParsedFrame(data).desc(abi.FORMAT_RGB_F32)[0]
    return fpx.token_lf_image(spec, int(d.global_scale))


@pytest.mark.parametrize("case", ["staggered", "unused", "tok2-mid", "tok3-start"])
def test_multi_pass_token_frames(ctx, case):
    """Shifted 2- and 3-pass token frames from their LF integers: groups with 0, 1 and 2 passes in one frame, and a
    group whose arrived pass 1 lies past its pass count."""
    if case == "staggered":
        spec, (data, cut) = P.spec_of("tok3"), P.staggered_case()
        assert set(j.PrefixParsedFrame(data[:cut]).passes.tolist()) == {0, 1, 2}
    elif case == "unused":
        spec, (data, cut) = P.spec_of("tok3"), P.unused_case()
    else:
        name, kind = case.split("-")
        spec, data = _token(name)
        cut = _cut(data, kind)
    gs.check_frames(ctx, [data], f"tokens {case}", cuts=[cut], lf_images=[_lf_image(spec, data)])


@pytest.mark.parametrize("name", ["tok_cc_lo", "tok_cc_hi", "tok_cc_zero"])
def test_token_lf_colour_correlation(ctx, name):
    """ytox_lf / ytob_lf at -128, 127 and 0 with other factors and bases, checked from the LF integers on: at the end
    of HfGlobal every group is the upsampled LF image; half way, decoded groups take it as their LLF."""
    spec, data = _token(name)
    lf = _lf_image(spec, data)
    for kind in ("start", "mid"):
        gs.check_frames(ctx, [data], f"{name} {kind}", headers=[spec["header"]], cuts=[_cut(data, kind)], lf_images=[lf])


FORMATS = [abi.FORMAT_RGB_U8, abi.FORMAT_RGBA_U8, abi.FORMAT_RGB_F32, abi.FORMAT_RGB_U16, abi.FORMAT_RGB_F16]
VIEW = {abi.FORMAT_RGB_U8: (np.uint8, 3), abi.FORMAT_RGBA_U8: (np.uint8, 4), abi.FORMAT_RGB_F32: (np.float32, 3),
        abi.FORMAT_RGB_U16: (np.uint16, 3), abi.FORMAT_RGB_F16: (np.uint16, 3)}


def _outputs(ctx, data, cut, fmts, what):
    """Each output format of data[:cut] against stage C of the GPU's filtered planes (check_output)."""
    whole = j.ParsedFrame(data)
    pf = j.PrefixParsedFrame(data[:cut])
    bx, (xyb,) = gs.run(ctx, [pf], abi.FORMAT_XYB_F32_PLANAR)
    bx.close()
    for fmt in fmts:
        fr = fp.Frame(whole.desc(fmt)[0])
        c, mc = fp.stage_c(fr, xyb.astype(np.float64))
        mc = np.where(fp.srgb_f32_overflow(fr, xyb), np.inf, mc)
        _, (raw,) = decode(ctx, [pf], fmt)
        dt, ch = VIEW[fmt]
        got = raw.view(dt).reshape(pf.height, pf.width, ch)
        fp.check_output(fmt, got, c, mc, fr.output_tf, fr.orientation, f"{what} format {fmt}")


@pytest.mark.parametrize("colour", [0, 1, 3])
def test_every_format(ctx, colour):
    """sRGB, linear and PQ output: RGB_U8, RGBA_U8, RGB_F32, RGB_U16, RGB_F16 (XYB_F32_PLANAR is stage B)."""
    data, cut = P.seam_case() if colour == 0 else (lambda d: (d, mid_cut(d)))(synth.encode_synthetic(600, 520, 410 + colour, colour=colour))
    _outputs(ctx, data, cut, FORMATS, f"colour {colour}")


@pytest.mark.parametrize("orientation", range(1, 9))
def test_every_orientation(ctx, orientation):
    make = lambda t: synth.encode_synthetic(600, 400, 420 + orientation, orientation=orientation, toc=t)  # noqa: E731
    data = P.permuted(make, "reverse")
    _outputs(ctx, data, mid_cut(data), [abi.FORMAT_RGB_U8], f"orientation {orientation}")


def test_corrupt_unused_section_is_ignored(ctx):
    """An arrived section past its group's pass count, its bytes flipped: the decode succeeds, the group's status is 0
    and the whole frame and a region are byte-identical to the same cut without the corruption."""
    data, cut = P.unused_case()
    off, ln = pr.hf_sections(data)
    assert off[1, 4] + ln[1, 4] <= cut and j.PrefixParsedFrame(data[:cut]).passes[4] == 0
    bad = bytearray(data[:cut])
    for i in range(int(off[1, 4]), int(off[1, 4] + ln[1, 4])):
        bad[i] ^= 0xA5
    region = (200, 200, 400, 300)  # group 4 (the middle one) and its neighbours
    want = [decode(ctx, [item])[1][0] for item in (j.PrefixParsedFrame(data[:cut]), (j.PrefixParsedFrame(data[:cut]), region))]
    for item in (j.PrefixParsedFrame(bytes(bad)), (j.PrefixParsedFrame(bytes(bad)), region)):
        b, (got,) = decode(ctx, [item], keep=True)
        status = b.stream_status(0)
        b.close()
        assert not np.asarray(status).any()
        assert np.array_equal(got, want.pop(0))
    gs.check_frames(ctx, [data], "unused section, clean", cuts=[cut], lf_images=[_lf_image(P.spec_of("tok3"), data)],
                    regions=[[region]])


def test_mixed_batch(ctx):
    """Partial prefixes with each (Gaborish, EPF) pair, a whole frame and a token frame from its LF integers in one
    batch, and regions of two of them: every frame meets its own float64 reference."""
    datas, cuts, lfs, regions = [], [], [], []
    for i, (gab, epf) in enumerate((g, e) for g in (0, 1) for e in range(4)):
        d = synth.encode_synthetic(600, 520, 430 + i, epf_iters=epf, gab=gab, colour=(0, 1, 3)[i % 3])
        datas.append(d)
        cuts.append(mid_cut(d) if i % 2 else pr.prefix_start(d))
        lfs.append(None)
        regions.append([(250, 240, 30, 40)] if i in (1, 6) else [])
    datas.append(synth.encode_synthetic(520, 512, 440))
    cuts.append(None)
    lfs.append(None)
    regions.append([])
    spec, d = _token("tok2")
    datas.append(d)
    cuts.append(mid_cut(d))
    lfs.append(_lf_image(spec, d))
    regions.append([(10, 250, 500, 20)])
    gs.check_frames(ctx, datas, "mixed prefix batch", cuts=cuts, lf_images=lfs, regions=regions)
