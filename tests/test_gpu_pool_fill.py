"""Outputs must not depend on what the device buffers held before a batch ran. Every device intermediate comes from a
pool of the context (batch_common.h) that is reused batch after batch, by both engines, and never cleared; the pool-fill
hook (JxgContext.set_pool_fill, jxg_context_set_pool_fill) writes one byte over all of them, and over the pinned staging
arena, before each run. 0xFF reads as an f32 NaN, as i32 -1 and as the block plan's "plan failed" nblk; 0x7F as an f32
of about 3.4e38 and a large positive i32. Each set below decodes on a new context without the hook, then on a context
filled with 0xFF and on one filled with 0x7F, and every byte must agree:

  (a) VarDCT: outputs, read_coeffs, read_xyb after the transforms (debug stop 2) and XYB_F32_PLANAR, on the token
      frames of test_vardct_ref in one batch per entropy route test_gpu_vardct_ref asserts (lean with and without the
      (4, 2, 0) form and the shared-memory context map, prefix, multi-pass / LZ77, all nineteen mixed), 8 lanes per
      warp and a two-pass frame of large varblocks (k_dequant_idct's CTA path adds the passes up in the planes); the
      header-field sets of test_gpu_header_fields (one batch per filter path); the custom dequantisation frames; the
      frames of test_gpu_f64_stages (all eight Gaborish / EPF pairs, one-pixel edge tiles, profiles 0-3) and its real
      fixtures plus the multi-pass progressive_ac; every output format at orientations 1-8. The float64 check (gpu_stages.check_frames) then runs on a poisoned context for one
      set per route: lean and prefix frames, an LZ77 frame, custom tables and header fields.
  (b) Modular: the token frames of test_modular_ref, test_modular_squeeze, test_modular_lz77 and
      test_modular_walk_table at 1, 2 and 4 lanes per warp, equal to the integer model, and the real Modular fixtures
      (lz77_flower takes the host-decoded-planes path) equal to the oracle.
  (c) errors: the decode errors of both engines, overlapping varblocks on each entropy route and one corrupt file per
      engine report the same code and first bad (frame, group); the valid frames of the batch keep their bytes.
  (d) one context without the hook, reused across five batches of both engines: each output equals the batch alone.
  (e) reruns: a rerun over pools filled with another byte gives the same device outputs.
  (f) batch composition: each frame of a batch of several routes, filter configurations and formats decodes to the
      same bytes alone, in the batch and in the reversed batch.
  (g) caller outputs pre-filled with the fill byte: every image sample is overwritten (the bytes agree under two
      prefills), device row padding is left alone; VarDCT, the Modular store and PipelinedDecoder.
  (h) the hook reaches the pools: after the entropy stage alone, read_xyb returns the fill pattern.

Subsets: the token frames run as six batches rather than nineteen single frames, since the route a batch takes is what
the kernels branch on; the output formats and orientations run on one 320x192 frame (test_gpu_output_stage's); the
float64 check runs once per route, not per set, because the bit equality with the new context carries the rest."""
import os

import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import test_gpu_vardct_ref as GV
from tests import test_vardct_ref as T

pytestmark = pytest.mark.gpu

FILLS = (0xFF, 0x7F)
U8, XYB = abi.FORMAT_RGB_U8, abi.FORMAT_XYB_F32_PLANAR


@pytest.fixture(scope="module")
def poisoned():
    """One context per fill byte, with the hook on."""
    import jxl_rs_b200 as j
    cs = {}
    for byte in FILLS:
        cs[byte] = j.JxgContext(0)
        cs[byte].set_pool_fill(byte)
    yield cs
    for c in cs.values():
        c.close()


def each_context(poisoned):
    """(label, context): a new context without the hook, then the poisoned ones."""
    import jxl_rs_b200 as j
    fresh = j.JxgContext(0)
    try:
        yield "new", fresh
        for byte, c in poisoned.items():
            yield hex(byte), c
    finally:
        fresh.close()


def _same(runs, what):
    """runs: [(label, list of arrays)]; every array equal, byte for byte, to the first run's."""
    label0, first = runs[0]
    for label, arrays in runs[1:]:
        assert len(arrays) == len(first), (what, label)
        for i, (a, b) in enumerate(zip(first, arrays)):
            a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
            assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), \
                f"{what}: item {i} differs between the {label0} context and the {label} context"


def _out_shape(pf, fmt):
    """(rows, row bytes) of a tight output of frame `pf` in `fmt`."""
    if fmt == XYB:
        return 3 * pf.info.coded_height, pf.info.coded_width * 4
    return pf.info.height, pf.info.width * abi.BYTES_PER_PIXEL[fmt]


def vardct(ctx, frames, fmts, debug_stop=0, prefill=0, pad=0, device=False, descs=None):
    """One batch over parsed `frames`, frame i into format fmts[i], outputs of `pad` extra bytes per row pre-filled
    with `prefill`. descs[i], when given and not None, replaces frame i's descriptor (Batch.add_desc). Returns the open
    batch, its entropy route, the error of wait() (None: none) and the whole output buffers as host arrays."""
    import torch
    import jxl_rs_b200 as j
    b = j.Batch(ctx, len(frames))
    if debug_stop:
        b.set_debug_stop(debug_stop)
    bufs = []
    for i, (pf, fmt) in enumerate(zip(frames, fmts)):
        rows, row = _out_shape(pf, fmt)
        buf = torch.full((rows, row + pad), prefill, dtype=torch.uint8, device="cuda" if device else "cpu")
        if not device:
            buf = buf.pin_memory()
        if descs and descs[i] is not None:
            d, hf, off, ln, n = descs[i]
            b.add_desc(d, hf, off, ln, n, buf.data_ptr(), row + pad, device)
        else:
            b.add(pf, buf.data_ptr(), row + pad, fmt, device)
        bufs.append(buf)
    b.run()
    route = b.entropy_stats()
    err = None
    try:
        b.wait()
    except abi.JxgError as e:
        err = e
    return b, route, err, [buf.cpu().numpy() for buf in bufs]


def _image(buf, pf, fmt):
    rows, row = _out_shape(pf, fmt)
    return buf[:rows, :row]


def vardct_taps(ctx, frames, fmts=None):
    """Coefficients and stage-A planes (debug stop 2), the outputs in `fmts` (default RGB_U8) and XYB_F32_PLANAR of
    one batch over `frames`, and the route of its entropy stage."""
    fmts = fmts or [U8] * len(frames)
    b, route, err, _ = vardct(ctx, frames, fmts, debug_stop=2)
    assert err is None, err
    taps = [b.read_coeffs(i) for i in range(len(frames))] + [b.read_xyb(i, 0) for i in range(len(frames))]
    b.close()
    for fm in (fmts, [XYB] * len(frames)):
        b, _, err, outs = vardct(ctx, frames, fm)
        b.close()
        assert err is None, err
        taps += [_image(o, pf, f) for o, pf, f in zip(outs, frames, fm)]
    return taps, route


def same_on_every_context(poisoned, datas, what, fmts=None, check=None):
    """(a): vardct_taps on each context agree; check(route, taps) runs on each."""
    import jxl_rs_b200 as j
    frames = [j.ParsedFrame(d) for d in datas]
    runs = []
    for label, ctx in each_context(poisoned):
        taps, route = vardct_taps(ctx, frames, fmts)
        if check:
            check(route, taps)
        runs.append((label, taps))
    _same(runs, what)


# ---------------------------------------------------------------- (a) VarDCT

# token frames of test_vardct_ref by the entropy route test_gpu_vardct_ref.ROUTES gives them
TOKEN_SETS = {
    "lean_420_smem": ["default_420", "qf15", "shapes_large", "thin", "flat", "ragged_tall_wide"],
    "lean_smem": ["one_block_context", "lf_x", "lf_y", "lf_b", "lf_all64", "entry_edges"],
    "lean_420_global": ["hist3", "hist_groups"],
    "fast": ["prefix"],
    "slow": ["orders", "passes11", "passes2_wrap", "lz77"],
    "mixed": T.CASES,
}


@pytest.mark.parametrize("name", list(TOKEN_SETS))
def test_token_frames_on_every_route(poisoned, name):
    names = TOKEN_SETS[name]
    models = [T.model(n) for n in names]
    groups = sum(f.num_groups for f, _ in models)
    kinds = {GV.ROUTES[n] for n in names}

    def check(route, taps):
        if len(kinds) == 1:
            GV._check_route(route, *next(iter(kinds)), groups)
        else:
            assert route["lean"] + route["fast"] + route["slow"] == groups, route
        for (f, _), c in zip(models, taps):
            assert np.array_equal(c, f.coeffs), name
    same_on_every_context(poisoned, [d for _, d in models], f"tokens {name}", check=check)


def multipass_large_frame():
    """Two passes over DCT128X128 and DCT64X64 varblocks, which k_dequant_idct's CTA path adds up in the planes
    themselves (the token frames' multi-pass varblocks all go through shared-memory tiles)."""
    from tests import vardct_ref as R
    rng = np.random.default_rng(128)
    xb = yb = 32
    vbs = T.tile(xb, yb, rng, T.MIXED, {(0, 0): [21], (16, 0): [21], (0, 16): [18], (8, 16): [18]})
    ps = [T.one_pass(shift=2, clusters=3), T.one_pass(shift=0, clusters=4, salt=5)]
    f = R.Frame(256, 256, vbs, T.lf_field(rng, xb, yb), R.BlockContextMap(), 1, ps, [0, 0])
    f.decode(T.chooser(17))
    assert f.error is None, f.error
    return f


def test_multipass_large_varblocks(poisoned):
    import synth
    f = multipass_large_frame()

    def check(route, taps):
        assert route["slow"] == 1, route
        assert np.array_equal(taps[0], f.coeffs)
    same_on_every_context(poisoned, [synth.encode_vardct_tokens(f.spec)], "two passes, large varblocks", check=check)


def test_eight_lanes_per_warp(poisoned):
    """Eight 4096 x 4096 frames (2048 lean streams) with three live contexts: the lean kernel runs 8 lanes per warp.
    Device outputs, compared on the device."""
    import torch
    import jxl_rs_b200 as j
    import synth
    pf = j.ParsedFrame(synth.encode_synthetic(4096, 4096, 88, 1.0, 2, 1, 1))
    want = None
    for label, ctx in each_context(poisoned):
        b = j.Batch(ctx, 8)
        outs = [torch.empty((4096, 4096, 3), dtype=torch.uint8, device="cuda") for _ in range(8)]
        for o in outs:
            b.add(pf, o.data_ptr(), 4096 * 3, U8, True)
        b.run()
        route = b.entropy_stats()
        b.wait()
        b.close()
        assert route["lean"] == 2048 and route["lean_S"] == 8, route
        for o in outs[1:]:
            assert torch.equal(o, outs[0]), label
        if want is None:
            want = outs[0]
        else:
            assert torch.equal(outs[0], want), label


def test_header_field_sets(poisoned):
    from tests import test_f64_header_fields as HF
    from tests import test_gpu_header_fields as HG
    for what, cases in (("vector", HG.VECTOR), ("scalar", HG.SCALAR), ("cfl", HG.CFL)):
        same_on_every_context(poisoned, [HF.written(c, n)[0] for n, c in cases], f"header fields {what}")


def test_custom_dequant_tables(poisoned):
    from tests import f64_quant as fq
    from tests import test_gpu_dequant_matrices as DQ
    datas = [DQ._frame(size, fq.profile4_encodings(es, modes), epf, gab, xq, bq)
             for size, es, modes, epf, gab, xq, bq in DQ.CASES]
    same_on_every_context(poisoned, datas, "custom dequant tables")


def test_filter_pairs_profiles_and_entropy_codes(poisoned):
    """test_gpu_f64_stages.SYNTHETIC (all eight Gaborish / EPF pairs, one-pixel edge tiles, profiles 0-3, a prefix
    frame, several output colour encodings) in one batch; then prefix and both LZ77 forms at profile 2."""
    import synth
    from tests import test_gpu_f64_stages as F
    same_on_every_context(poisoned, [F._synthetic(c) for c in F.SYNTHETIC], "f64 stage frames")
    same_on_every_context(poisoned, [synth.encode_synthetic(600, 520, 31 + e, 1.0, 2, 1, 2, entropy=e) for e in (1, 2, 3)],
                          "prefix and LZ77")


def test_real_fixtures(poisoned, golden_dir):
    from tests import test_gpu_f64_stages as F
    names = F.FIXTURES + ["progressive_ac"]
    datas = [open(os.path.join(golden_dir, "jxl", n + ".jxl"), "rb").read() for n in names]
    same_on_every_context(poisoned, datas, "real VarDCT fixtures")


def test_every_format_and_orientation(poisoned):
    """test_gpu_output_stage.decode at every format and orientation, host and device outputs with padded rows."""
    from tests import test_gpu_output_stage as OS
    pf = OS._frame(320, 192, 52, 1.0, 2, 1)
    runs = []
    for label, ctx in each_context(poisoned):
        got = []
        for fmt in OS.FORMATS:
            for o in range(1, 9):
                for device in (False, True):
                    samples, b, _ = OS.decode(ctx, pf, fmt, {"orientation": o}, pad=16, device=device)
                    b.close()
                    got.append(samples)
        runs.append((label, got))
    _same(runs, "formats and orientations")


def test_float64_check_on_poisoned_pools(poisoned):
    """gpu_stages.check_frames, every run of it on a poisoned context: lean frames with one-pixel edge tiles and a
    prefix frame, an LZ77 frame, custom tables, a header-field set."""
    import synth
    from tests import f64_quant as fq
    from tests import test_f64_header_fields as HF
    from tests import test_gpu_dequant_matrices as DQ
    from tests import test_gpu_f64_stages as F
    from tests import test_gpu_header_fields as HG
    from tests.gpu_stages import check_frames
    c_ff, c_7f = poisoned[0xFF], poisoned[0x7F]
    check_frames(c_ff, [F._synthetic(F.SYNTHETIC[i]) for i in (5, 6, 7)], "poisoned 0xff: lean + prefix")
    check_frames(c_7f, [synth.encode_synthetic(300, 280, 33, 1.0, 1, 0, 1, entropy=2)], "poisoned 0x7f: LZ77")
    encs = fq.profile4_encodings(1, {})
    check_frames(c_7f, [DQ._frame(DQ.ALL_TABLES[0], encs)], "poisoned 0x7f: custom tables", [encs])
    name, case = HG.VECTOR[-1]
    data, header = HF.written(case, name)
    check_frames(c_ff, [data], f"poisoned 0xff: header {name}", headers=[header])


# ---------------------------------------------------------------- (b) Modular

def modular_sets():
    """(label, model-or-None, file) of the Modular token frames; the model is an object with .u8 and planes."""
    from tests import test_modular_lz77 as L
    from tests import test_modular_ref as MR
    from tests import test_modular_squeeze as S
    from tests import test_modular_walk_table as W
    out = []
    for n in MR.CASES:
        f, d = MR.model(n)
        out.append((f"ref {n}", MR.model_planes(f), f.u8, d))
    for n in S.CASES:
        if n != "local_squeeze":
            f, d = S.model(n)
            out.append((f"squeeze {n}", S.T.model_planes(f), f.u8, d))
    for n in L.TOKEN_CASES:
        for mode in (1, 2):
            f, d, _ = L.token_frame(n, mode)
            out.append((f"lz77 {n} {mode}", L.model_planes(f), f.u8, d))
    for n in W.CASES:
        for it, d in W.items(n):
            out.append((f"walk {it.label}", MR.model_planes(it.frame), it.frame.u8, d))
    for n in sorted(W.LZ77_CASES):
        for it, d, _ in W.lz77_items(n):
            out.append((f"walk lz77 {it.label}", MR.model_planes(it.frame), it.frame.u8, d))
    return out


def test_modular_token_frames(poisoned):
    from tests.gpu_modular import gpu_decode
    for label, planes, u8, data in modular_sets():
        runs = []
        for ctx_label, ctx in each_context(poisoned):
            got = []
            for lanes in (1, 2, 4):
                (out,), (p,) = gpu_decode(ctx, [data], lanes)
                assert np.array_equal(np.asarray(p).reshape(-1), planes.reshape(-1).astype(np.int32)), (label, ctx_label, lanes)
                assert np.array_equal(out, u8), (label, ctx_label, lanes)
                got += [out, p]
            runs.append((ctx_label, got))
        _same(runs, label)


MODULAR_FIXTURES = ["green_queen_modular_e3.jxl", "grayscale_public_university.jxl", "issue865_large_toc.jxl",
                    "3x3_srgb_lossless.jxl", "lz77_flower.jxl", "tree_max_property_20.jxl"]


def test_modular_real_files(poisoned, golden_dir):
    from tests import oracle_binding as ob
    from tests.gpu_modular import gpu_decode
    for name in MODULAR_FIXTURES:
        data = open(os.path.join(golden_dir, "jxl", name), "rb").read()
        ref, ref_planes = ob.decode_modular_file(data, planes=True)
        runs = []
        for label, ctx in each_context(poisoned):
            (out,), (planes,) = gpu_decode(ctx, [data], 4)
            assert np.array_equal(planes, ref_planes) and np.array_equal(out, ref), (name, label)
            runs.append((label, [out, planes]))
        _same(runs, name)


# ---------------------------------------------------------------- (c) errors

def _error_runs(poisoned, run):
    """run(ctx) -> (JxgError or None, arrays of the valid frames); the error's code and message (which names the first
    bad frame and group) and the arrays must agree on every context."""
    runs, errs = [], []
    for label, ctx in each_context(poisoned):
        err, arrays = run(ctx)
        assert err is not None, label
        errs.append((err.code, str(err)))
        runs.append((label, arrays))
    assert len(set(errs)) == 1, errs
    _same(runs, errs[0][1])
    return errs[0]


@pytest.mark.parametrize("case", ["invalid_num_nonzeros", "residual_nonzeros", "histogram_index"])
def test_vardct_decode_errors(poisoned, case):
    """The refused frame between two valid frames: the error names frame 1, and frames 0 and 2 keep their bytes."""
    import jxl_rs_b200 as j
    import synth
    bad, good, kind = T.refusal_pairs()[case]
    good, bad = good(), bad()
    frames = [j.ParsedFrame(synth.encode_vardct_tokens(x.spec)) for x in (good, bad, good)]

    def run(ctx):
        b, _, err, outs = vardct(ctx, frames, [U8] * 3)
        coeffs = [b.read_coeffs(0), b.read_coeffs(2)]
        b.close()
        assert np.array_equal(coeffs[0], good.coeffs)
        return err, [outs[0], outs[2]] + coeffs
    code, msg = _error_runs(poisoned, run)
    assert code == {"InvalidNumNonZeros": -5, "EndOfBlockResidualNonZeros": -6, "InvalidHistogramIndex": -4}[kind]
    assert "frame 1 group" in msg, msg


@pytest.mark.parametrize("entropy", [0, 1, 2], ids=["lean", "fast", "slow"])
def test_overlapping_varblocks(poisoned, entropy):
    """test_gpu_pipeline.overlapping_varblocks on one frame of a batch of three (the same file unmutated around it)."""
    import jxl_rs_b200 as j
    import synth
    from tests.test_gpu_pipeline import overlapping_varblocks
    w, h = 300, 200
    pf = j.ParsedFrame(synth.encode_synthetic(w, h, 9, 0.5, 2, 1, 1, entropy=entropy))
    d = pf.desc(U8)
    keep = overlapping_varblocks(d[0], w, h)  # noqa: F841 - keeps replacement buffers alive

    def run(ctx):
        b, _, err, outs = vardct(ctx, [pf] * 3, [U8] * 3, descs=[None, d, None])
        b.close()
        return err, [outs[0], outs[2]]
    code, msg = _error_runs(poisoned, run)
    assert code == -8 and "frame 1 group" in msg, msg  # JXG_ERR_INVALID_TRANSFORM


def test_corrupt_vardct_file(poisoned, golden_dir):
    """green_queen_vardct_e3 with its HF bytes flipped (test_gpu_parity), after a valid frame."""
    import jxl_rs_b200 as j
    good = open(os.path.join(golden_dir, "jxl", "green_queen_vardct_e3.jxl"), "rb").read()
    data = bytearray(good)
    for i in range(len(data) - 3000, len(data) - 2000):
        data[i] ^= 0x5a
    frames = [j.ParsedFrame(good), j.ParsedFrame(bytes(data))]

    def run(ctx):
        b, _, err, outs = vardct(ctx, frames, [U8] * 2)
        b.close()
        return err, [outs[0]]
    _, msg = _error_runs(poisoned, run)
    assert "frame 1 group" in msg, msg


@pytest.mark.parametrize("fault", [1, 2], ids=["copy_first", "length_overflow"])
def test_modular_lz77_errors(poisoned, fault):
    from tests import test_modular_lz77 as L
    from tests.gpu_modular import gpu_decode
    good_frame, good, _ = L.token_frame("ans_tree", 2, lz=L.ERROR_LZ)
    _, bad, _ = L.token_frame("ans_tree", 2, fault=(fault, 4), lz=L.ERROR_LZ)
    for lanes in (1, 4):
        def run(ctx):
            (out, _), (planes, _), err = gpu_decode(ctx, [good, bad], lanes, expect_error=True)
            assert np.array_equal(out, good_frame.u8)
            return err, [out, planes]
        code, msg = _error_runs(poisoned, run)
        assert code == -10 and "frame 1 group 2" in msg, msg


@pytest.mark.parametrize("source", ["writer", "green_queen_modular_e3.jxl"])
def test_corrupt_modular_file(poisoned, golden_dir, source):
    """A Modular file with bytes flipped inside its last group sections, after its intact twin (one geometry, one
    global transform structure)."""
    import synth
    from tests.gpu_modular import gpu_decode
    if source == "writer":
        good = synth.encode_modular(600, 520, 9, 6, 0, 1)
        bad = bytearray(good)
        bad[-2000] ^= 0x5A  # test_gpu_modular.test_corrupt_modular_stream_reports_group
    else:
        good = open(os.path.join(golden_dir, "jxl", source), "rb").read()
        bad = bytearray(good)
        for i in range(len(bad) - 600, len(bad) - 500):
            bad[i] ^= 0x5A

    def run(ctx):
        (out, _), (planes, _), err = gpu_decode(ctx, [good, bytes(bad)], 2, expect_error=True)
        return err, [out, planes]
    code, msg = _error_runs(poisoned, run)
    assert code != -20 and "frame 1 group" in msg, msg  # a stream error, never JXG_ERR_CUDA


def test_modular_refusals(poisoned):
    """The palette-range and local-tree refusals of test_gpu_modular_ref: the same error on every context."""
    import synth
    from tests import test_modular_ref as MR
    from tests.gpu_modular import gpu_decode
    frames = [MR._refusal_frame([("leaf", 5, 0, 0, 0)], False, **kw) for _, kw in MR.PALETTE_REFUSALS]
    frames += [MR._refusal_frame([("leaf", 5, 0, 0, 0)], False, groups={0: {"tree": bad}}) for _, bad, _ in MR.REFUSALS]
    for f in frames:
        data = synth.encode_modular_tokens(f.spec)
        errs = set()
        for _, ctx in each_context(poisoned):
            with pytest.raises(abi.JxgError) as e:
                gpu_decode(ctx, [data])
            errs.add((e.value.code, str(e.value)))
        assert len(errs) == 1, errs


# ---------------------------------------------------------------- (d) one context, five batches

def _modular(ctx, files, lanes=2):
    """Outputs and planes of one ModularBatch over `files`."""
    from tests.gpu_modular import gpu_decode
    outs, planes = gpu_decode(ctx, files, lanes)
    return outs + planes


def test_reused_context_without_the_hook(golden_dir):
    """Five batches of both engines on one context without the hook; each equals the same batch on a new context."""
    import jxl_rs_b200 as j
    import synth
    from tests import f64_quant as fq
    from tests import test_gpu_dequant_matrices as DQ
    from tests import test_gpu_output_stage as OS
    encs = fq.profile4_encodings(3)
    big = [synth.encode_synthetic(1030, 770, 61, 0.8, 2, 1, 2, entropy=2), T.model("passes11")[1], T.model("passes2_wrap")[1],
           DQ._frame(DQ.ALL_TABLES[1], encs), synth.encode_synthetic(2048, 1024, 62, 1.0, 3, 1, 3)]
    big_frames = [j.ParsedFrame(d) for d in big]
    small = [j.ParsedFrame(synth.encode_synthetic(200, 136, 63 + i, 1.0, 1, 0, 1, entropy=1)) for i in range(2)]
    pf = OS._frame(257, 131, 64, 1.0, 0, 0)
    modular_a = [synth.encode_modular(1030, 770, 65, 6, 1, 2)]
    modular_b = [synth.encode_modular(700, 530, 66, 6, 0, 3), synth.encode_modular(700, 530, 67, 6, 0, 2)]

    def vardct_u8(ctx, frames):
        return vardct_taps(ctx, frames)[0]

    def oriented(ctx):
        got = []
        for fmt, o in ((abi.FORMAT_RGB_F32, 6), (abi.FORMAT_RGB_U16, 3)):
            samples, b, _ = OS.decode(ctx, pf, fmt, {"orientation": o}, pad=8, device=True)
            b.close()
            got.append(samples)
        return got
    steps = [("large VarDCT", lambda c: vardct_u8(c, big_frames)), ("Modular WP + Squeeze", lambda c: _modular(c, modular_a)),
             ("small prefix VarDCT", lambda c: vardct_u8(c, small)), ("orientation / format / filter", oriented),
             ("Modular again", lambda c: _modular(c, modular_b, 4))]
    shared = j.JxgContext(0)
    try:
        for what, step in steps:
            got = step(shared)
            alone = j.JxgContext(0)
            try:
                want = step(alone)
            finally:
                alone.close()
            _same([("new", want), ("reused", got)], what)
    finally:
        shared.close()


# ---------------------------------------------------------------- (e) reruns

def test_vardct_rerun_over_refilled_pools():
    import torch
    import jxl_rs_b200 as j
    import synth
    from tests import f64_quant as fq
    from tests import test_gpu_dequant_matrices as DQ
    frames = [j.ParsedFrame(d) for d in (synth.encode_synthetic(600, 520, 71, 1.0, 2, 1, 2, entropy=2), T.model("passes11")[1],
                                         DQ._frame(DQ.ALL_TABLES[0], fq.profile4_encodings(4)), T.model("default_420")[1])]
    ctx = j.JxgContext(0)
    try:
        ctx.set_pool_fill(0xFF)
        outs = [torch.zeros((pf.info.height, pf.info.width * 3), dtype=torch.uint8, device="cuda") for pf in frames]
        b = j.Batch(ctx, len(frames))
        for pf, o in zip(frames, outs):
            b.add(pf, o.data_ptr(), o.shape[1], U8, True)
        b.run()
        b.wait()
        first = [o.clone() for o in outs] + [torch.from_numpy(b.read_coeffs(i)) for i in range(len(frames))]
        ctx.set_pool_fill(0x7F)
        for o in outs:
            o.fill_(0x7F)
        b.rerun_device()
        b.wait()
        second = [o.clone() for o in outs] + [torch.from_numpy(b.read_coeffs(i)) for i in range(len(frames))]
        b.close()
    finally:
        ctx.close()
    for i, (x, y) in enumerate(zip(first, second)):
        assert torch.equal(x.cpu(), y.cpu()), i


def test_modular_rerun_over_refilled_pools():
    import torch
    import jxl_rs_b200 as j
    import synth
    files = [synth.encode_modular(1030, 770, 72, 6, 1, 2), synth.encode_modular(1030, 770, 73, 6, 1, 1)]
    frames = [j.ModularParsedFrame(f) for f in files]
    ctx = j.JxgContext(0)
    try:
        ctx.set_pool_fill(0xFF)
        outs = [torch.zeros((fr.height, fr.width * 3), dtype=torch.uint8, device="cuda") for fr in frames]
        b = j.ModularBatch(ctx, 2)
        for fr, o in zip(frames, outs):
            b.add(fr, o.data_ptr(), o.shape[1], True)
        b.run()
        b.wait()
        first = [o.clone() for o in outs] + [torch.from_numpy(b.read_planes(i)) for i in range(2)]
        ctx.set_pool_fill(0x7F)
        for o in outs:
            o.fill_(0x7F)
        b.rerun_device()
        b.wait()
        second = [o.clone() for o in outs] + [torch.from_numpy(b.read_planes(i)) for i in range(2)]
        b.close()
    finally:
        ctx.close()
    for i, (x, y) in enumerate(zip(first, second)):
        assert torch.equal(x.cpu(), y.cpu()), i
    assert np.array_equal(first[0].cpu().numpy().reshape(770, 1030, 3), synth.modular_source(1030, 770, 72))


# ---------------------------------------------------------------- (f) batch composition and order

def test_batch_composition_and_order(poisoned):
    """Lean, prefix, LZ77 and multi-pass frames with different filter configurations, each in its own format: every
    frame decodes to the same bytes alone, in the batch and in the reversed batch, on a new and a poisoned context."""
    import jxl_rs_b200 as j
    import synth
    from tests import test_gpu_f64_stages as F
    datas = [T.model("default_420")[1], F._synthetic(F.SYNTHETIC[5]), synth.encode_synthetic(300, 200, 81, 1.0, 3, 1, 1, entropy=2),
             F._synthetic(F.SYNTHETIC[4]), T.model("passes2_wrap")[1], F._synthetic(F.SYNTHETIC[6]),
             synth.encode_synthetic(520, 512, 82, 1.0, 2, 1, 1)]
    frames = [j.ParsedFrame(d) for d in datas]
    fmts = [U8, abi.FORMAT_RGB_F32, abi.FORMAT_RGBA_U8, abi.FORMAT_RGB_U16, abi.FORMAT_RGB_F16, XYB, U8]
    alone_ctx = j.JxgContext(0)
    try:
        alone = []
        for pf, fmt in zip(frames, fmts):
            b, _, err, (o,) = vardct(alone_ctx, [pf], [fmt])
            b.close()
            assert err is None, err
            alone.append(_image(o, pf, fmt))
    finally:
        alone_ctx.close()
    n = len(frames)
    for label, ctx in [("new", None)] + [(hex(k), c) for k, c in poisoned.items()]:
        own = ctx is None
        ctx = ctx or j.JxgContext(0)
        try:
            for order in (list(range(n)), list(range(n))[::-1]):
                b, _, err, outs = vardct(ctx, [frames[i] for i in order], [fmts[i] for i in order])
                b.close()
                assert err is None, err
                got = [None] * n
                for k, i in enumerate(order):
                    got[i] = _image(outs[k], frames[i], fmts[i])
                _same([("alone", alone), (f"{label} batch order {order[:2]}...", got)], "batch composition")
        finally:
            if own:
                ctx.close()


# ---------------------------------------------------------------- (g) caller outputs start as poison

@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_vardct_outputs_start_as_poison(poisoned, device):
    """Outputs with 12 bytes of row padding pre-filled with 0x00 and with the fill byte: the image bytes agree (every
    sample was written) and, on the device, the padding still holds the prefill."""
    import jxl_rs_b200 as j
    from tests import test_gpu_f64_stages as F
    from tests import test_gpu_output_stage as OS
    frames = [j.ParsedFrame(F._synthetic(F.SYNTHETIC[i])) for i in (0, 6, 9)]
    for byte, ctx in poisoned.items():
        for fmt in OS.FORMATS:
            images = []
            for prefill in (0, byte):
                b, _, err, outs = vardct(ctx, frames, [fmt] * len(frames), prefill=prefill, pad=12, device=device)
                b.close()
                assert err is None, err
                for pf, o in zip(frames, outs):
                    if device:
                        assert (o[:, _out_shape(pf, fmt)[1]:] == prefill).all(), (fmt, "row padding overwritten")
                images.append([_image(o, pf, fmt) for o, pf in zip(outs, frames)])
            _same([("prefill 0", images[0]), (f"prefill {byte:#x}", images[1])], f"format {fmt}")


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_modular_outputs_start_as_poison(poisoned, device):
    import torch
    import jxl_rs_b200 as j
    import synth
    sizes = [(513, 300, 91), (64, 48, 92)]
    for byte, ctx in poisoned.items():
        for w, h, seed in sizes:
            fr = j.ModularParsedFrame(synth.encode_modular(w, h, seed, 0, 1, 0))
            for prefill in (0, byte):
                stride = w * 3 + 5
                buf = torch.full((h, stride), prefill, dtype=torch.uint8, device="cuda" if device else "cpu")
                if not device:
                    buf = buf.pin_memory()
                b = j.ModularBatch(ctx, 2)
                b.add(fr, buf.data_ptr(), stride, device)
                b.run()
                b.wait()
                b.close()
                host = buf.cpu().numpy()
                assert np.array_equal(host[:, :w * 3].reshape(h, w, 3), synth.modular_source(w, h, seed)), (w, prefill)
                if device:
                    assert (host[:, w * 3:] == prefill).all(), (w, "row padding overwritten")


def test_pipelined_decoder_with_poisoned_contexts():
    """PipelinedDecoder with the hook on in each of its contexts, into pre-filled pinned outputs with 7 bytes of row
    padding: every image equals the batch decoded alone on a new context into rows of the same stride (a tight row
    of a 4-byte multiple would let the fused filter's interior tiles take its vector store path, whose last bits may
    differ from the scalar path's)."""
    import torch
    import jxl_rs_b200 as j
    import synth
    sets = [[synth.encode_synthetic(300 + 8 * i, 200 + 16 * k, 95 + 10 * k + i, 0.6, 2, 1, 1, entropy=k % 3)
             for i in range(3)] for k in range(4)]
    ctx = j.JxgContext(0)
    try:
        want = []
        for files in sets:
            frames = [j.ParsedFrame(f) for f in files]
            b, _, err, outs = vardct(ctx, frames, [U8] * len(frames), pad=7)
            b.close()
            assert err is None, err
            want.append([_image(o, pf, U8) for o, pf in zip(outs, frames)])
    finally:
        ctx.close()
    dec = j.PipelinedDecoder(0, depth=2, staging_threads=2)
    try:
        for c, byte in zip(dec.ctxs, FILLS):
            c.set_pool_fill(byte)
        bufs = []
        for k, files in enumerate(sets):
            row = []
            for f in files:
                fr = j.ParsedFrame(f)
                row.append(torch.full((fr.height, fr.width * 3 + 7), FILLS[k % 2], dtype=torch.uint8).pin_memory())
            bufs.append(row)
            dec.submit(files, [(b.data_ptr(), b.shape[1]) for b in row])
        dec.drain()
    finally:
        dec.close()
    for k, (w_set, b_set) in enumerate(zip(want, bufs)):
        for i, (w, b) in enumerate(zip(w_set, b_set)):
            assert np.array_equal(b.numpy()[:, :w.shape[1]], w), (k, i)


# ---------------------------------------------------------------- (h) the hook reaches the pools

def test_hook_fills_the_planes(poisoned):
    """Stopped after the entropy stage, the transforms never wrote the planes: read_xyb returns the fill pattern. And
    the hook refuses a byte outside -1..255."""
    import jxl_rs_b200 as j
    import synth
    pf = j.ParsedFrame(synth.encode_synthetic(300, 200, 99, 1.0, 2, 1, 1))
    for byte, ctx in poisoned.items():
        b, _, err, _ = vardct(ctx, [pf], [U8], debug_stop=1)
        assert err is None, err
        planes = b.read_xyb(0, 0)
        b.close()
        assert (planes.view(np.uint32) == byte * 0x01010101).all(), hex(byte)
    c = j.JxgContext(0)
    try:
        for bad in (-2, 256):
            with pytest.raises(abi.JxgError):
                c.set_pool_fill(bad)
        c.set_pool_fill(0)
        c.set_pool_fill(-1)
    finally:
        c.close()
