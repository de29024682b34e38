"""Entropy schedules that only very large batches reach on the device's own SM count, reached with small batches through
the SM budget hook (JxgContext.set_sm_budget), each one asserted through the schedule taps (Batch.entropy_schedule,
Batch.stream_status) so that a change of the scheduler cannot quietly drop the coverage:

  (a) batch.cc schedule_lean restated in Python and compared with the tap over frame counts (more frames than CTAs
      too), streams per frame (1, S, S + 1, 256) and budgets (1, 2, 7, the device's), with its invariants;
  (b) every k_entropy_lean instance ((4, 2, 0) or not x context map in shared memory or not x 4 or 8 lanes per warp), the
      8-lane ones also with queued streams, bit for bit against tests/vardct_ref.py, on new and poisoned contexts. Four
      lanes per warp never queue: the schedule goes to 8 lanes before it queues streams;
  (c) k_entropy_fast at 1, 2, 4 and 8 streams per warp, its warps holding lanes of different frames, beside lean and
      slow streams in the same batch;
  (d) lanes that end a failed stream and then take a good one: every kind of group failure, each group's status, the
      first bad (frame, group) of wait() and the good groups' coefficients; and failing lanes beside good ones in the
      warps of k_entropy_fast;
  (e) pixels that do not depend on the schedule: budget 1 against the device's own count, whole frames and regions;
  (f) the Modular decode queue and the grid-stride grids of the Modular transforms at budget 1.

The restatement itself, on the shapes the scheduler is designed around, runs without a GPU."""
import contextlib
import ctypes as C
import math
import os

import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import test_vardct_ref as T
from tests import vardct_ref as R

gpu = pytest.mark.gpu
U8, F32 = abi.FORMAT_RGB_U8, abi.FORMAT_RGB_F32
STATUS = {"nnz": -5, "residual": -6, "hist": -4, "width": -2, "overlap": -8}  # JXG_ERR_* of each group failure
BIG = [18, 19, 20, 5, 8, 9, 10, 11, 4]  # 64x64 .. 16x16 varblocks (and DCT8 where none fits): few blocks per group
CFGS = [(4, 2, 0), (0, 0, 0), (3, 1, 1), (5, 2, 1)]


# ---------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------
def schedule_lean(counts, sms, live=1):
    """batch.cc schedule_lean: counts[f] lean streams of frame f (0: none), `sms` SMs, `live` contexts on the device ->
    (S, [(lanes, ctas)] per frame, grid). Each frame's warps take S lanes (the last one fewer) and are padded to whole
    CTAs of 4 warps; the grid must fit one resident wave of 6 CTAs per SM. Denser packing goes first to 8 lanes per
    warp, then to ceil(count / per_lane) lanes rounded up to a multiple of S (per_lane *= 1.3 in float32) for at most
    12 attempts, and stops once every frame with lean streams is down to one CTA."""
    total = sum(counts)
    if not total:
        return None
    max_ctas = sms * 6
    S = 8 if live >= 3 and total >= 2048 else 4
    per_lane = np.float32(1.0)
    for _ in range(12):
        sched = []
        for c in counts:
            if not c:
                sched.append((0, 0))
                continue
            lanes = int(math.ceil(np.float32(c) / per_lane))
            lanes = min(c, (lanes + S - 1) // S * S)
            warps = (lanes + S - 1) // S
            sched.append((lanes, (warps + 3) // 4))
        grid = sum(ct for _, ct in sched)
        if grid <= max_ctas or all(ct == 1 for (_, ct), c in zip(sched, counts) if c):
            break
        if S < 8:
            S = 8
        else:
            per_lane = np.float32(per_lane * np.float32(1.3))
    return S, sched, grid


def fast_S(n, sms):
    """batch.cc schedule_fast: streams per warp of k_entropy_fast for n streams."""
    per = (n + sms * 16 - 1) // (sms * 16)
    return 0 if not n else 1 if per <= 1 else 2 if per <= 2 else 4 if per <= 4 else 8


def test_restatement_on_the_designed_shapes():
    # budget 1 (6 CTAs): one 256-group frame, three 81-group frames, seven 9-group frames
    assert schedule_lean([256], 1) == (8, [(152, 5)], 5)
    assert schedule_lean([81] * 3, 1) == (8, [(64, 2)] * 3, 6)
    assert schedule_lean([9] * 7, 1) == (4, [(9, 1)] * 7, 7)  # one CTA per frame already: nothing is queued
    assert schedule_lean([40] * 4, 1) == (8, [(32, 1)] * 4, 4)
    # 132 SMs (792 CTAs): 64 frames of 3840 x 2160 (135 groups) fit at 4 lanes per warp
    assert schedule_lean([135] * 64, 132) == (4, [(135, 9)] * 64, 576)
    # more frames than CTAs: the grid stops at one CTA per frame
    assert schedule_lean([40] * 1000, 132) == (8, [(32, 1)] * 1000, 1000)
    assert schedule_lean([16] * 800, 132) == (4, [(16, 1)] * 800, 800)
    assert schedule_lean([9] * 800, 132) == (4, [(9, 1)] * 800, 800)
    # three live contexts and 2048 streams or more: 8 lanes per warp from the start
    assert schedule_lean([256] * 8, 132, live=3) == (8, [(256, 8)] * 8, 64)
    assert schedule_lean([256] * 8, 132, live=2)[0] == 4
    assert fast_S(2112, 132) == 1 and fast_S(2113, 132) == 2 and fast_S(2560, 132) == 2 and fast_S(8449, 132) == 8


# ---------------------------------------------------------------------------------------------------------------
# token-level model frames
# ---------------------------------------------------------------------------------------------------------------
def group_of(f, bx, by):
    return (by // 32) * f.xg + bx // 32


def last_varblocks(f):
    """(by, bx) of the last varblock of each group in raster order of their top-left blocks."""
    last = {}
    for bx, by, _, _ in f.varblocks:
        g = group_of(f, bx, by)
        last[g] = max(last.get(g, (-1, -1)), (by, bx))
    return last


def group_chooser(seed, f, cap_of, fail):
    """Nonzero counts up to cap_of(group), their nonzeros within the first 4 * cap slots; fail[group] puts that group's
    failure in the last channel (B) of its last varblock: "nnz" one nonzero too many, "residual" a nonzero count the
    block does not use up, "width" a coefficient one past the device's entry width (the model decodes it)."""
    rng = np.random.default_rng(seed)
    last = last_varblocks(f)

    def choose(ev):
        g, nb, nc, shift = ev["g"], ev["num_blocks"], ev["num_coeffs"], ev["shift"]
        room = nc - nb
        kind = fail.get(g)
        if kind in ("nnz", "residual", "width") and ev["c"] == 2 and (ev["by"], ev["bx"]) == last[g]:
            if kind == "nnz":
                return room + 1, []
            if kind == "residual":
                return 2, [0] * (room - 1) + [3]
            return 1, [1 << (31 - (nc.bit_length() - 1))]
        cap = min(room, cap_of(g))
        nz = int(rng.integers(0, cap + 1))
        if not nz:
            return 0, []
        pos = np.sort(rng.choice(min(room, 4 * cap), nz, replace=False))
        vals = [0] * (int(pos[-1]) + 1)
        lim = max(1, 40 >> shift)
        for p in pos:
            vals[int(p)] = int(rng.integers(1, lim + 1)) * (1 if rng.random() < 0.5 else -1)
        return nz, vals
    return choose


_MODELS = {}


def model(key, w, h, seed, choices=BIG, cfgs=None, clusters=4, nh=1, prefix=False, shift=0, cap_of=lambda g: 6,
          fail=None, log_alpha=6):
    """(Frame, file bytes, expected status per group) of a single-pass token-level frame, cached under `key` (each
    caller's seed is its own). fail:
    {group: kind}; "hist" writes the group's histogram index as num_histograms (nh must not be a power of two) and
    "overlap" is applied to the descriptor (overlap_groups), so the model decodes both groups as good ones."""
    if key not in _MODELS:
        import synth
        fail = fail or {}
        rng = np.random.default_rng(seed)
        xb, yb = (w + 7) // 8, (h + 7) // 8
        vbs = T.tile(xb, yb, rng, choices)
        groups = ((w + 255) // 256) * ((h + 255) // 256)
        hist = [int(x) for x in rng.integers(0, nh, groups)]
        p = T.one_pass(shift=shift, clusters=clusters, cfgs=cfgs, prefix=prefix, log_alpha=log_alpha, salt=seed % 7)
        f = R.Frame(w, h, vbs, T.lf_field(rng, xb, yb), R.BlockContextMap(), nh, [p], hist)
        f.decode(group_chooser(seed, f, cap_of, fail), per_group=True)
        spec = f.spec
        for g, kind in fail.items():
            if kind == "hist":
                assert nh & (nh - 1), "an index past the count needs a count that is not a power of two"
                spec["sections"][g] = (nh, spec["sections"][g][1])
        status = np.zeros(groups, np.int32)
        for g in range(groups):
            if f.group_errors[g] is not None:
                status[g] = {"InvalidNumNonZeros": -5, "EndOfBlockResidualNonZeros": -6}[f.group_errors[g]]
            elif g in fail:
                status[g] = STATUS[fail[g]]
        assert [g for g in range(groups) if status[g]] == sorted(fail), (key, status)
        _MODELS[key] = (f, synth.encode_vardct_tokens(spec), status)
    return _MODELS[key]


def overlap_groups(d, w, h, groups):
    """test_gpu_pipeline.overlapping_varblocks on descriptor d, kept only in `groups`; returns the buffers to keep."""
    from tests.test_gpu_pipeline import overlapping_varblocks
    xb, yb, xg = (w + 7) // 8, (h + 7) // 8, (w + 255) // 256
    orig = C.string_at(d.transform_map, xb * yb)
    keep = overlapping_varblocks(d, w, h)
    for by in range(yb):
        for bx in range(xb):
            if (by // 32) * xg + bx // 32 not in groups:
                keep[0][by * xb + bx] = orig[by * xb + bx]
    return keep


def strip(groups, seed, **kw):
    """A frame of `groups` groups in one row, 16 pixels high, its last group ragged."""
    return model(("strip", groups, seed), groups * 256 - 5, 16, seed, choices=T.MIXED, **kw)


def grid36(seed, **kw):
    """A 6 x 6 group frame whose right and bottom groups are ragged."""
    return model(("grid36", seed), 1380, 1340, seed, **kw)


# ---------------------------------------------------------------------------------------------------------------
# device runs
# ---------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def context(budget=0, fill=-1, extra=0):
    """A new context with the SM budget and pool fill set; `extra` more live contexts beside it."""
    import jxl_rs_b200 as j
    cs = [j.JxgContext(0) for _ in range(1 + extra)]
    try:
        cs[0].set_sm_budget(budget)
        if fill >= 0:
            cs[0].set_pool_fill(fill)
        yield cs[0]
    finally:
        for c in cs:
            c.close()


def run(ctx, items, fmt=U8, coeffs=True, debug_stop=0, stride_pad=0):
    """One batch of items (ParsedFrame, descriptor tuple or None, region or None). Returns the schedule tap, the entropy
    stats, the JxgError of wait() (None if it succeeded), each whole frame's group status and coefficients, and the
    output bytes."""
    import torch
    import jxl_rs_b200 as j
    bpp = abi.BYTES_PER_PIXEL[fmt]
    b = j.Batch(ctx, len(items))
    outs, shapes = [], []
    try:
        for pf, desc, region in items:
            h, w = (pf.height, pf.width) if region is None else (region[3], region[2])
            stride = w * bpp + stride_pad
            o = torch.empty(h * stride, dtype=torch.uint8).pin_memory()
            outs.append(o)
            shapes.append((h, w * bpp))  # the pixels of each row, without the padding the decode leaves as it was
            if desc is None:
                b.add(pf, o.data_ptr(), stride, fmt, False, region)
            else:
                d, hf, off, ln, n = desc
                b.add_desc(d, hf, off, ln, n, o.data_ptr(), stride, False)
                b.frames.append(pf)
        if debug_stop:
            b.set_debug_stop(debug_stop)
        b.run()
        err = None
        try:
            b.wait()
        except abi.JxgError as e:
            err = e
        whole = [i for i, it in enumerate(items) if it[2] is None]
        res = {"sched": b.entropy_schedule(), "stats": b.entropy_stats(), "err": err,
               "status": {i: b.stream_status(i) for i in whole},
               "coeffs": {i: b.read_coeffs(i) for i in whole} if coeffs else {},
               "outs": [o.numpy().reshape(-1, o.numel() // len_rows)[:, :w_bytes].copy()
                        for o, (len_rows, w_bytes) in zip(outs, shapes)]}
    finally:
        b.close()
    return res


def check_schedule(res, counts, sms, live=1):
    """The tap against the restatement, and the invariants of the schedule."""
    sc = res["sched"]
    want = schedule_lean(counts, sms, live)
    got = [(fr["lanes"], fr["ctas"]) for fr in sc["frames"]]
    assert [fr["count"] for fr in sc["frames"]] == list(counts)
    assert (sc["lean_S"], got, sc["lean_ctas"]) == want, (counts, sms, sc, want)
    S = sc["lean_S"]
    for fr in sc["frames"]:
        assert fr["lanes"] <= fr["count"] and (fr["lanes"] % S == 0 or fr["lanes"] == fr["count"]), fr
    assert sum(fr["ctas"] for fr in sc["frames"]) == sc["lean_ctas"]
    assert sc["lean_lanes"] == sum(fr["lanes"] for fr in sc["frames"]) and sc["lean_count"] == sum(counts)
    # every queued stream taken once: one pull per queued stream, one empty pull per lane
    assert [fr["pulls"] for fr in sc["frames"]] == list(counts) and sc["lean_pulls"] == sum(counts), sc
    return S, sum(fr["count"] - fr["lanes"] for fr in sc["frames"])


def parsed(data):
    import jxl_rs_b200 as j
    return j.ParsedFrame(data)


def device_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_budget_argument():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    try:
        for n in (1, 7, 0):
            c.set_sm_budget(n)
        with pytest.raises(abi.JxgError) as e:
            c.set_sm_budget(-1)
        assert e.value.code == -22
    finally:
        c.close()
    lib = abi.load_library()
    assert lib.jxg_context_set_sm_budget(None, 1) == -22


@gpu
def test_schedule_equals_restatement():
    """Tiny frames of 1, 4, 5, 8, 9 and 256 groups, in batches of up to 800 frames, at budgets 1, 2, 7 and the device's
    own: the tap equals the restatement frame by frame, and every group decodes."""
    sms = device_sms()
    sizes = {1: model("one", 8, 8, 1, choices=T.MIXED)}
    for n in (4, 5, 8, 9, 256):
        sizes[n] = strip(n, 10 + n, cap_of=lambda g: 2)
    frames = {n: (parsed(v[1]), v[0]) for n, v in sizes.items()}
    sets = [[1], [1] * 7, [1] * 13, [5] * 7, [4, 5, 8, 9], [9] * 7, [8] * 3 + [9] * 4, [256], [256, 9, 1], [9] * 50,
            [5] * 60]
    cases = [(budget, s) for budget in (1, 2, 7, 0) for s in sets] + [(0, [1] * 800), (0, [9] * 800)]
    queued_seen = eight_seen = 0
    for budget, counts in cases:
        with context(budget) as ctx:
            res = run(ctx, [(frames[n][0], None, None) for n in counts], coeffs=False, debug_stop=1)
        S, queued = check_schedule(res, counts, budget or sms)
        assert res["err"] is None and all(not st.any() for st in res["status"].values())
        queued_seen += queued > 0
        eight_seen += S == 8
    assert queued_seen and eight_seen
    # three live contexts and 2,048 streams: 8 lanes per warp on the device's own count
    with context(0, extra=2) as ctx:
        res = run(ctx, [(frames[1][0], None, None)] * 2100, coeffs=False, debug_stop=1)
    assert check_schedule(res, [1] * 2100, sms, live=3)[0] == 8


INSTANCES = [(a420, smem) for a420 in (True, False) for smem in (True, False)]


def instance_frame(a420, smem):
    """A 36-group frame on the lean route: (4, 2, 0) in every cluster or not; one histogram (its context map fits
    the shared staging area) or three (it does not)."""
    return grid36(100 + 2 * a420 + smem, cfgs=None if a420 else CFGS, nh=1 if smem else 3, cap_of=lambda g: 3 + g % 5)


@gpu
@pytest.mark.parametrize("a420,smem", INSTANCES, ids=[f"{'420' if a else 'any'}-{'smem' if s else 'global'}"
                                                      for a, s in INSTANCES])
def test_every_lean_instance(a420, smem):
    """One, three and four copies of the frame at budgets that give 4 lanes per warp, 8 lanes, and 8 lanes with
    queued streams; on a new context and on one whose pools are filled with 0xFF."""
    f, data, _ = instance_frame(a420, smem)
    pf = parsed(data)
    sms = device_sms()
    for copies, budget, S, queue in ((1, 0, 4, False), (3, 1, 8, False), (4, 1, 8, True)):
        for fill in (-1, 0xFF):
            with context(budget, fill) as ctx:
                res = run(ctx, [(pf, None, None)] * copies)
            st = res["stats"]
            assert (st["lean"], st["lean_all_420"], st["lean_ctx_smem"]) == (36 * copies, a420, smem), st
            got_S, queued = check_schedule(res, [36] * copies, budget or sms)
            assert got_S == S and (queued > 0) == queue, res["sched"]
            assert res["err"] is None
            for i in range(copies):
                assert not res["status"][i].any()
                assert np.array_equal(res["coeffs"][i], f.coeffs), (copies, budget, fill, i)


def fast_frames():
    """Prefix-coded frames with different pass tables: 4, 2, 6, 3 and 5 clusters, different hybrid-uint configurations,
    one and two histograms, few and many nonzeros (shorter and longer codes); 5, 7, 11, 15 and 31 groups."""
    return [
        strip(5, 51, prefix=True, cfgs=[(4, 2, 0), (0, 0, 0), (1, 1, 0), (4, 1, 3)]),
        strip(7, 52, prefix=True, clusters=2),
        strip(11, 53, prefix=True, cfgs=[(4, 2, 0), (2, 1, 0), (5, 2, 1), (0, 0, 0), (4, 0, 0), (6, 3, 3)],
              cap_of=lambda g: 40),
        strip(15, 54, prefix=True, cfgs=[(0, 0, 0), (4, 2, 0), (2, 0, 1)], cap_of=lambda g: 12),
        strip(31, 55, prefix=True, nh=2, clusters=5, cap_of=lambda g: 1 + g % 9),
    ]


@gpu
def test_fast_kernel_lanes_per_warp():
    """At budget 1 (a wave of 16 warps) 12, 23, 38 and 69 fast streams take 1, 2, 4 and 8 streams per warp; none is a
    multiple of its S, so warps hold lanes of two frames; a lean and a two-pass frame share each batch."""
    fr = fast_frames()
    lean = strip(9, 60)
    slow_f, slow_data = T.model("passes2_wrap")
    items = [(parsed(d), None, None) for _, d, _ in fr]
    lean_item, slow_item = (parsed(lean[1]), None, None), (parsed(slow_data), None, None)
    for k, S in ((2, 1), (3, 2), (4, 4), (5, 8)):
        n = sum(f.num_groups for f, _, _ in fr[:k])
        assert n % S or S == 1
        for fill in (-1, 0xFF):
            with context(1, fill) as ctx:
                res = run(ctx, [lean_item] + items[:k] + [slow_item])
            assert res["err"] is None
            assert res["sched"]["fast_S"] == S == fast_S(n, 1), res["sched"]
            assert (res["stats"]["lean"], res["stats"]["fast"], res["stats"]["slow"]) == (9, n, slow_f.num_groups)
            models = [lean[0]] + [f for f, _, _ in fr[:k]] + [slow_f]
            for i, f in enumerate(models):
                assert not res["status"][i].any()
                assert np.array_equal(res["coeffs"][i], f.coeffs), (S, fill, i)


def failing_frame(kind):
    """grid36 with every group failing except four full ones, which are the shortest: the failing groups write many
    nonzeros before their failure at the last varblock, the good ones at most 2 per channel."""
    good = {0, 8, 15, 22}
    fail = {g: kind for g in range(36) if g not in good}
    if kind == "overlap":  # the corner group's 50 overlapping varblocks fit its coefficient area, which the block
        fail[35] = "nnz"   # plan checks, so it is made to fail another way
    return grid36(200 + sorted(STATUS).index(kind), nh=3 if kind == "hist" else 1, fail=fail,
                  cap_of=lambda g: 2 if g in good else 60), good


def _descs(pf, kind, w, h, groups):
    if kind != "overlap":
        return None, None
    d = pf.desc(U8)
    return d, overlap_groups(d[0], w, h, groups)


def check_failures(res, models, frames_status):
    """Every group's status, the first bad (frame, group) of wait() and the good groups' coefficients."""
    first = None
    for i, (f, status) in enumerate(zip(models, frames_status)):
        assert np.array_equal(res["status"][i], status), (i, res["status"][i], status)
        bad = np.flatnonzero(status)
        if first is None and len(bad):
            first = (i, int(bad[0]), int(status[bad[0]]))
        for g in np.flatnonzero(status == 0):
            assert np.array_equal(res["coeffs"][i][g], f.coeffs[g]), (i, g)
    assert res["err"] is not None and res["err"].code == first[2], res["err"]
    assert f"frame {first[0]} group {first[1]}" in str(res["err"]), (str(res["err"]), first)


@gpu
@pytest.mark.parametrize("kind", sorted(STATUS))
def test_lean_lane_after_a_failed_stream(kind):
    """Four copies at budget 1: 8 lanes per warp, 32 lanes per frame; the 32 failing groups start, the 4 good ones are
    queued and each is taken by a lane that has just ended a failed stream."""
    (f, data, status), good = failing_frame(kind)
    pf = parsed(data)
    d, keep = _descs(pf, kind, f.width, f.height, {g for g in range(36) if status[g] == -8})  # noqa: F841
    lens = np.ctypeslib.as_array(C.cast(pf.desc(U8)[3], C.POINTER(C.c_uint32)), (36,))
    assert lens[sorted(good)].max() < np.delete(lens, sorted(good)).min(), lens
    for fill in (-1, 0xFF):
        with context(1, fill) as ctx:
            res = run(ctx, [(pf, d, None)] * 4)
        S, queued = check_schedule(res, [36] * 4, 1)
        assert S == 8 and [fr["lanes"] for fr in res["sched"]["frames"]] == [32] * 4
        check_failures(res, [f] * 4, [status] * 4)


@gpu
def test_fast_lanes_beside_failed_ones():
    """A prefix frame of 36 groups at budget 1 (4 streams per warp) whose groups fail in every way or decode, in turn,
    beside a frame of good groups: failing and good lanes share warps."""
    kinds = [None, "nnz", None, "residual", "width", None, "hist", "overlap"]
    fail = {g: kinds[g % 8] for g in range(36) if kinds[g % 8]}
    f, data, status = grid36(300, prefix=True, nh=3, fail=fail, cap_of=lambda g: 8)
    g_f, g_data, g_status = strip(7, 52, prefix=True, clusters=2)
    pf = parsed(data)
    d, keep = _descs(pf, "overlap", f.width, f.height, {g for g, k in fail.items() if k == "overlap"})  # noqa: F841
    for fill in (-1, 0xFF):
        with context(1, fill) as ctx:
            res = run(ctx, [(parsed(g_data), None, None), (pf, d, None)])
        assert res["sched"]["fast_S"] == 4 and res["stats"]["fast"] == 43, res
        check_failures(res, [g_f, f], [g_status, status])


def _fixtures(golden_dir):
    from tests import test_gpu_f64_stages as F
    return [open(os.path.join(golden_dir, "jxl", n + ".jxl"), "rb").read() for n in F.FIXTURES + ["progressive_ac"]]


@gpu
@pytest.mark.parametrize("fmt", [U8, F32], ids=["u8", "f32"])
def test_pixels_do_not_depend_on_the_schedule(golden_dir, fmt):
    """The full pipeline at budget 1 (queued streams) and at the device's own count gives the same bytes: the four
    instance frames and the real VarDCT fixtures in one batch, then regions of the instance frames."""
    items = [(parsed(instance_frame(*k)[1]), None, None) for k in INSTANCES]
    items += [(parsed(d), None, None) for d in _fixtures(golden_dir)]
    regions = [(pf, None, (7, 5, pf.width - 20, pf.height - 13)) for pf, _, _ in items[:4]] * 2
    for batch in (items, regions):
        got = {}
        for budget in (1, 0):
            with context(budget) as ctx:
                got[budget] = run(ctx, batch, fmt, coeffs=False, stride_pad=16)
            assert got[budget]["err"] is None
        sc = got[1]["sched"]
        assert sc["lean_S"] == 8 and any(fr["lanes"] < fr["count"] for fr in sc["frames"]), sc
        for a, b in zip(got[1]["outs"], got[0]["outs"]):
            assert np.array_equal(a, b)


@gpu
def test_modular_at_budget_one():
    """The token-level Modular frames, the LZ77 and Squeeze sets at budget 1 with 1, 2 and 4 lanes per warp equal the
    integer model. A batch of a plain and an LZ77 frame of 96 groups each runs both decode launches, whose lanes (at
    most 32 warps each) take queued streams at 1 and 2 lanes per warp, and its transform and store grids stride (16
    CTAs of 256 threads per job); the frames are lossless, so both decode to their source."""
    import synth
    from tests import test_modular_lz77 as L
    from tests import test_modular_ref as MT
    from tests import test_modular_squeeze as S
    from tests.gpu_modular import gpu_decode
    with context(1) as ctx:
        for name in MT.CASES:
            frame, data = MT.model(name)
            for lanes in (1, 2, 4):
                (out,), (planes,) = gpu_decode(ctx, [data], lanes)
                assert np.array_equal(np.asarray(planes).reshape(-1), MT.model_planes(frame).reshape(-1).astype(np.int32))
                assert np.array_equal(out, frame.u8), name
        for name in L.TOKEN_CASES:
            for mode in (1, 2):
                frame, data, _ = L.token_frame(name, mode)
                for lanes in (1, 2, 4):
                    (out,), (planes,), st = gpu_decode(ctx, [data], lanes, lz77_stats=True)
                    assert st["lz77_streams"] > 0
                    assert np.array_equal(np.asarray(planes).reshape(-1), L.model_planes(frame).reshape(-1).astype(np.int32))
                    assert np.array_equal(out, frame.u8), (name, mode)
        for name in S.CASES:
            if name == "local_squeeze":
                continue
            frame, data = S.model(name)
            for lanes in (1, 2, 4):
                (out,), (planes,) = gpu_decode(ctx, [data], lanes)
                assert np.array_equal(np.asarray(planes).reshape(-1), S.T.model_planes(frame).reshape(-1).astype(np.int32))
                assert np.array_equal(out, frame.u8), name
        w, h = 3072, 2048
        src = L.flat_picture(w, h, 3)
        files = [synth.encode_modular(w, h, 7, source=src, lz77=0), synth.encode_modular(w, h, 7, source=src, lz77=1)]
        for lanes in (1, 2, 4):
            outs, _, st = gpu_decode(ctx, files, lanes, lz77_stats=True)
            assert st["lz77_streams"] == 96, st
            for o in outs:
                assert np.array_equal(o, src)
