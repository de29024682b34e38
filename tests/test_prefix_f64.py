"""The prefix decode's float64 side and its test files, on the CPU (tests/f64_prefix.py):

  - permuted TOCs (synth's `toc`): the oracle decodes a permuted file to the coefficients and RGB_U8 bytes of the
    unpermuted one, and prefix_ref.group_passes agrees with the prefix parse at every section boundary of it;
  - the float64 LF image of token-level frames, from their LF integers and the ytox_lf / ytob_lf written, against the
    front end's LF planes, with both branches of the smoothing gate taken;
  - the frames and cuts test_gpu_prefix_f64.py runs, which must reach a zero-pass group with a decoded right and
    bottom neighbour and an arrived section past its group's pass count."""
import numpy as np
import pytest

import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from tests import f64_pipeline as fp
from tests import f64_prefix as fpx
from tests import oracle_binding as ob
from tests import prefix_ref as pr
from tests import vardct_ref as R


# ---------------------------------------------------------------------------------------------------------------------
# Token-level frames with chosen LF integers
# ---------------------------------------------------------------------------------------------------------------------
def smooth_and_rough_lf(rng, xb, yb):
    """LF integers whose left third is linear ramps (the smoothing's full blend, gap 0.5), middle third ramps with +-1
    steps (partial blends) and right third noise (the gate closed, factor 0)."""
    yy, xx = np.mgrid[0:yb, 0:xb]
    lf = np.stack([(xx // 4 - 5), (yy // 3 + xx // 5 - 10), (10 - yy // 4)]).astype(np.int64)
    mid = (xx >= xb // 3) & (xx < 2 * xb // 3)
    lf = lf + mid * rng.integers(-1, 2, (3, yb, xb))
    rough = xx >= 2 * xb // 3
    return np.where(rough, rng.integers(-40, 41, (3, yb, xb)), lf)


def token_case(name):
    """(spec, what) of a token-level frame: a model frame decoded with test_vardct_ref's chooser, then its spec."""
    from tests import test_vardct_ref as T
    rng = np.random.default_rng(sum(map(ord, name)) * 31)
    w, h, shifts, color = {
        "tok2": (600, 560, [2, 0], None),
        "tok3": (600, 560, [3, 1, 0], None),
        "tok_cc_lo": (520, 300, [0], {"ytox_lf": -128, "ytob_lf": -128}),
        "tok_cc_hi": (520, 300, [1, 0], {"ytox_lf": 127, "ytob_lf": 127, "factor": (1, 0), "base_x": 0xB400}),
        "tok_cc_zero": (300, 520, [0], {"ytox_lf": 0, "ytob_lf": 0, "factor": (2, 40), "base_b": 0x3A00}),
    }[name]
    xb, yb = (w + 7) // 8, (h + 7) // 8
    ps = [T.one_pass(shift=s, clusters=3 + i, salt=i) for i, s in enumerate(shifts)]
    ng = ((w + 255) // 256) * ((h + 255) // 256)
    f = R.Frame(w, h, T.tile(xb, yb, rng, T.MIXED), smooth_and_rough_lf(rng, xb, yb), R.BlockContextMap(), 1, ps,
                [0] * (len(shifts) * ng))
    f.decode(T.chooser(len(name) + 7, vmax=30))
    assert f.error is None, f.error
    spec = f.spec
    if color is not None:
        spec = dict(spec, header={"color": color})
    return spec


TOKEN_NAMES = ["tok2", "tok3", "tok_cc_lo", "tok_cc_hi", "tok_cc_zero"]
_SPECS = {}


def spec_of(name):
    if name not in _SPECS:
        _SPECS[name] = token_case(name)
    return _SPECS[name]


def frame_counts(data):
    fr = j.ParsedFrame(data)
    d = fr.desc(abi.FORMAT_RGB_F32)[0]
    xb, yb = (d.width + 7) // 8, (d.height + 7) // 8
    return ((xb + 255) // 256) * ((yb + 255) // 256), fr.info.num_groups, fr.info.num_passes


def permuted(make, kind):
    """make(toc) -> file bytes; the file with the named permutation of its sections."""
    nlf, ng, npass = frame_counts(make(None))
    return make(fpx.toc_permutation(kind, nlf, ng, npass))


# ---------------------------------------------------------------------------------------------------------------------
# The files and cuts of the GPU module
# ---------------------------------------------------------------------------------------------------------------------
def section_end(data, p, g):
    off, ln = pr.hf_sections(data)
    return int(off[p, g] + ln[p, g])


def synth_file(w, h, seed, toc=None, **kw):
    return synth.encode_synthetic(w, h, seed, toc=toc, **kw)


def seam_case():
    """1100 x 700 (5 x 3 groups) with the groups stored in reverse: cut after group 6, so groups 0-5 have no pass and
    lie left of and above decoded ones; group 5, the first of the middle row, has decoded right (6) and bottom (10)
    neighbours."""
    data = permuted(lambda t: synth_file(1100, 700, 301, t), "reverse")
    return data, section_end(data, 0, 6)


def unused_case():
    """A 3-pass token frame, each group's pass 1 stored before its pass 0: cut after group 4's pass 1, so its pass 1
    has arrived and is unused (k = 0), groups 0-3 have all three passes and 5-8 none."""
    data = permuted(lambda t: synth.encode_vardct_tokens(dict(spec_of("tok3"), toc=t)), "pass1_first")
    return data, section_end(data, 1, 4)


def staggered_case():
    """A 3-pass token frame stored pass 0 of groups 0-7, pass 1 of groups 0-4, then the rest in order: cut before group
    8's pass 0, so one frame holds groups with 2 passes (0-4), 1 pass (5-7) and none (8)."""
    spec = spec_of("tok3")
    nlf, ng, npass = frame_counts(synth.encode_vardct_tokens(spec))
    head = list(range(2 + nlf))
    hf = lambda p, g: fpx.hf_index(nlf, ng, p, g)  # noqa: E731
    body = [hf(0, g) for g in range(ng - 1)] + [hf(1, g) for g in range(5)]
    rest = [i for i in range(2 + nlf + npass * ng) if i not in head + body]
    data = synth.encode_vardct_tokens(dict(spec, toc=fpx.perm_from_stored(head + body + rest)))
    return data, section_end(data, 1, 4)


def test_cases_reach_their_shapes():
    """The two shapes no writer order reached: a zero-pass group with a decoded right and bottom neighbour, and an
    arrived section past its group's pass count; and pass counts 0, 1 and 2 in one frame."""
    data, cut = seam_case()
    k = j.PrefixParsedFrame(data[:cut]).passes
    xg = (1100 + 255) // 256
    kk = k.reshape(-1, xg)
    both = [(gy, gx) for gy in range(kk.shape[0] - 1) for gx in range(xg - 1)
            if kk[gy, gx] == 0 and kk[gy, gx + 1] > 0 and kk[gy + 1, gx] > 0]
    assert both, kk
    data, cut = unused_case()
    off, ln = pr.hf_sections(data)
    k = j.PrefixParsedFrame(data[:cut]).passes
    arrived = off + ln <= cut
    unused = [(p, g) for p in range(off.shape[0]) for g in range(off.shape[1]) if arrived[p, g] and p >= k[g]]
    assert (1, 4) in unused and k[4] == 0, (unused, k)
    data, cut = staggered_case()
    assert set(j.PrefixParsedFrame(data[:cut]).passes.tolist()) == {0, 1, 2}


# ---------------------------------------------------------------------------------------------------------------------
# Permuted TOCs
# ---------------------------------------------------------------------------------------------------------------------
PERMUTED = [("synth", "reverse"), ("tok2", "reverse"), ("tok3", "reverse"), ("tok3", "interleaved"),
            ("tok3", "pass1_first"), ("tok2", "pass1_first")]


def _maker(src):
    if src == "synth":
        return lambda t: synth_file(700, 600, 311, t, profile=3)
    return lambda t: synth.encode_vardct_tokens(dict(spec_of(src), toc=t))


@pytest.mark.parametrize("src,kind", PERMUTED)
def test_permuted_file_decodes_as_the_unpermuted(src, kind):
    make = _maker(src)
    plain, perm = make(None), permuted(make, kind)
    assert plain != perm and len(plain) > len(perm) - 64
    out_a, taps_a = ob.decode_file(plain, abi.FORMAT_RGB_U8, taps=True)
    out_b, taps_b = ob.decode_file(perm, abi.FORMAT_RGB_U8, taps=True)
    assert np.array_equal(taps_a["coeffs"], taps_b["coeffs"])
    assert np.array_equal(out_a, out_b)
    # the sections are where the permutation put them: stored order differs from logical order
    off, _ = pr.hf_sections(perm)
    assert not (np.diff(off.reshape(-1)) > 0).all()


@pytest.mark.parametrize("src,kind", PERMUTED)
def test_group_passes_at_every_boundary_of_permuted_files(src, kind):
    data = permuted(_maker(src), kind)
    off, ln = pr.hf_sections(data)
    start = pr.prefix_start(data)
    ends = sorted({int(v) for v in (off + ln).ravel()} | {int(v) for v in off.ravel()})
    for e in ends:
        for cut in (e - 1, e, e + 1):
            if start <= cut <= len(data):
                assert np.array_equal(j.PrefixParsedFrame(data[:cut]).passes, pr.group_passes(off, ln, cut)), cut


def test_single_toc_entry_is_refused():
    with pytest.raises(RuntimeError, match="single TOC entry"):
        synth.encode_synthetic(200, 200, 5, toc=[0])
    with pytest.raises(RuntimeError, match="wrong size"):
        synth.encode_synthetic(300, 200, 5, toc=[0, 1, 2])


# ---------------------------------------------------------------------------------------------------------------------
# The float64 LF image
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", TOKEN_NAMES)
def test_lf_image_against_the_front_end(name):
    spec = spec_of(name)
    data = synth.encode_vardct_tokens(spec)
    pf = j.ParsedFrame(data)
    d = pf.desc(abi.FORMAT_RGB_F32)[0]
    host = fp.Frame(d, header=spec.get("header")).lf
    lf, mag, gate = fpx.token_lf_image(spec, int(d.global_scale))
    ratio = fp.check("A", host, lf, mag * (fpx.K_LF / fp.BOUND_K["A"]), f"{name} LF image")
    print(name, "largest err/(2^-24 M) of the LF image:", round(ratio, 2), "K_LF", fpx.K_LF)
    assert ratio <= fpx.K_LF
    inner = gate[~np.isnan(gate)]
    assert (inner == 0).any() and (inner > 0).any() and ((inner > 0) & (inner < 1)).any(), name


def test_lf_image_pins_the_colour_correlation():
    """The helper takes ytox_lf / ytob_lf from the header written: the same frame with the fields moved by one is
    outside the bound in X and B (and, through the smoothing gate the channels share, in some Y samples too)."""
    spec = spec_of("tok_cc_hi")
    d = j.ParsedFrame(synth.encode_vardct_tokens(spec)).desc(abi.FORMAT_RGB_F32)[0]
    host = fp.Frame(d, header=spec["header"]).lf
    moved = dict(spec, header={"color": dict(spec["header"]["color"], ytox_lf=126, ytob_lf=126)})
    lf, mag, _ = fpx.token_lf_image(moved, int(d.global_scale))
    bad = np.abs(host - lf) > fpx.K_LF * fp.EPS * mag + 1e-9
    assert bad[0].mean() > 0.5 and bad[2].mean() > 0.5


def test_smoothing_gate_is_continuous():
    """The gate's bound relies on max(0, 3 - 4 gap) having no jump: samples either side of gap = 0.75 give nearly
    equal outputs."""
    lf = np.zeros((3, 3, 3))
    dcf = np.array([1.0, 1.0, 1.0])
    outs = []
    for d in (0.75 / (1 - fpx.W_CENTER) - 1e-9, 0.75 / (1 - fpx.W_CENTER) + 1e-9):
        x = lf.copy()
        x[0, 1, 1] = d  # |mc - sm| = d (1 - W_CENTER)
        out, _, f = fpx.smooth_lf_f64(x, np.zeros_like(x), dcf)
        outs.append(out[0, 1, 1])
        assert abs(f[1, 1]) < 1e-8
    assert abs(outs[0] - outs[1]) < 1e-7
