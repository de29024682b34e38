"""The transform kernels take their varblocks from the block plan's class partition (k_block_plan: BatchDev::cls_n /
cls_list). Checked here:

  * the partition itself, read through jxg_batch_read_transform_plan, against a restatement from each frame's transform
    map: per-class counts and entry lists (ordinal, position, transform type) of every group, including groups with empty classes, a group holding one
    DCT256X256 only, and frames whose block plan fails (every count 0);
  * XYB_F32_PLANAR and RGB_U8 outputs byte-identical between a context scheduled for one SM and one scheduled for the
    device's own count, on the token frames of vardct_ref.py, synthetic frames of profiles 0-4 (every transform class,
    the 128 / 256 families and the 8x8 specials), a two-pass DCT128X128 / DCT64X64 frame, ragged frame sizes and the
    real fixtures;
  * the planes after dequant + IDCT (debug stop 2) within the float64 stage-A bound of tests/gpu_stages.py."""
import os

import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import f64_pipeline as fp
from tests import test_vardct_ref as T

pytestmark = pytest.mark.gpu

U8, XYB = abi.FORMAT_RGB_U8, abi.FORMAT_XYB_F32_PLANAR
COV_X, COV_Y = fp.COV_X, fp.COV_Y

# The partition restated: bucket of each transform type (classes 0..2 split by type, in the kernels' order), then the
# class of each bucket. Class 3: the other types of at most 4 x 4 blocks; class 4: larger varblocks.
TYPE_ORDER = {0: 0, 3: 1, 12: 2, 13: 3, 6: 4, 7: 5, 4: 6}
BUCKET_CLASS = [0, 0, 0, 0, 1, 1, 2, 3, 4]


def bucket(t):
    if t in TYPE_ORDER:
        return TYPE_ORDER[t]
    return 7 if COV_X[t] <= 4 and COV_Y[t] <= 4 else 8


def restated_plan(tmap):
    """tmap: [yb, xb] u8 transform map. Per group in raster order: (counts[5], entries class after class), or None when
    the block plan fails (a type >= 27, or varblocks whose coefficients overflow the group's 65536). Entry of a varblock:
    its ordinal in the group's raster order | bx << 10 | by << 15 (first block inside the group) | type << 20."""
    yb, xb = tmap.shape
    plans = []
    for gy in range(0, yb, 32):
        for gx in range(0, xb, 32):
            sub = tmap[gy:gy + 32, gx:gx + 32]
            firsts = [(int(v) & 127, i % sub.shape[1], i // sub.shape[1]) for i, v in enumerate(sub.ravel()) if v >= 128]
            if any(t >= 27 for t, _, _ in firsts) or sum(COV_X[t] * COV_Y[t] * 64 for t, _, _ in firsts) > 65536:
                plans.append(None)
                continue
            buckets = [[] for _ in range(9)]
            for seq, (t, bx, by) in enumerate(firsts):
                buckets[bucket(t)].append(seq | bx << 10 | by << 15 | t << 20)
            counts = [0] * 5
            for b, lst in enumerate(buckets):
                counts[BUCKET_CLASS[b]] += len(lst)
            plans.append((counts, [s for lst in buckets for s in lst]))
    return plans


def transform_map(pf):
    import ctypes as C
    d = pf.desc(U8)[0]
    xb, yb = (pf.info.coded_width + 7) // 8, (pf.info.coded_height + 7) // 8
    return np.frombuffer(C.string_at(d.transform_map, xb * yb), np.uint8).reshape(yb, xb)


def check_plan(batch, f, tmap, what):
    """The device partition of frame f equals the restatement. Returns the restated plans."""
    plans = restated_plan(tmap)
    counts, seqs = batch.transform_plan(f, len(plans))
    assert counts.shape[0] == len(plans), what
    for g, p in enumerate(plans):
        if p is None:
            assert not counts[g].any(), f"{what}: group {g}: failed plan with classes {counts[g].tolist()}"
            continue
        want_n, want_seq = p
        assert counts[g, :5].tolist() == want_n and not counts[g, 5:].any(), \
            f"{what}: group {g}: class counts {counts[g].tolist()}, restated {want_n}"
        assert seqs[g, :len(want_seq)].tolist() == want_seq, f"{what}: group {g}: class lists differ"
    return plans


# ---------------------------------------------------------------------------------------------------------------- sets

def _synthetic(w, h, seed, profile, **kw):
    import synth
    return synth.encode_synthetic(w, h, seed, 1.0, 2, 1, profile, **kw)


def big_only_frame():
    """512 x 256 token frame: group 0 is one DCT256X256 (only the CTA class), group 1 a random mix of the 8x8 to 32x32
    types."""
    import synth
    from tests import vardct_ref as R
    rng = np.random.default_rng(256)
    xb, yb = 64, 32
    vbs = T.tile(xb, yb, rng, T.MIXED, {(0, 0): [24]})
    f = R.Frame(512, 256, vbs, T.lf_field(rng, xb, yb), R.BlockContextMap(), 1, [T.one_pass(clusters=4)], [0, 0])
    f.decode(T.chooser(19))
    assert f.error is None, f.error
    return synth.encode_vardct_tokens(f.spec)


def frame_sets(golden_dir):
    """name -> (list of file bytes, the header each frame was written with for the float64 stage-A check, or None: no
    float64 check)."""
    import synth
    from tests import f64_header as fh
    from tests import test_gpu_pool_fill as PF
    from tests import test_gpu_f64_stages as F
    fixtures = [open(os.path.join(golden_dir, "jxl", n + ".jxl"), "rb").read() for n in F.FIXTURES]
    sets = {
        "tokens": [T.model(n)[1] for n in T.CASES],
        "profiles": [_synthetic(520, 512, 40 + p, p) for p in range(5)],
        "two_pass_large": [synth.encode_vardct_tokens(PF.multipass_large_frame().spec), big_only_frame()],
        "ragged": [_synthetic(w, h, 50 + k, p) for k, (w, h, p) in
                   enumerate([(1, 1, 0), (9, 17, 4), (129, 97, 1), (263, 131, 2), (777, 513, 3), (300, 1030, 4)])],
    }
    out = {k: (v, [None] * len(v)) for k, v in sets.items()}
    out["fixtures"] = (fixtures, [fh.OPSIN_INVERSE_FIXTURE if n == "opsin_inverse" else None for n in F.FIXTURES])
    # progressive_ac (3.4 MP, IDENTITY / DCT2X2 / AFV, two passes): over the f64 budget per case, outputs only
    out["progressive_ac"] = ([open(os.path.join(golden_dir, "jxl", "progressive_ac.jxl"), "rb").read()], None)
    return out


def decode(ctx, frames, fmt, debug_stop=0):
    """One batch; returns (batch, host outputs); the caller closes the batch."""
    from tests import gpu_stages as G
    return G.run(ctx, frames, fmt, debug_stop)


@pytest.fixture(scope="module")
def contexts():
    """(one-SM schedule, the device's own count)."""
    import jxl_rs_b200 as j
    one, own = j.JxgContext(0), j.JxgContext(0)
    one.set_sm_budget(1)
    yield one, own
    one.close()
    own.close()


@pytest.mark.parametrize("name", ["tokens", "profiles", "two_pass_large", "ragged", "fixtures", "progressive_ac"])
def test_plan_outputs_and_stage_a(contexts, golden_dir, name):
    import jxl_rs_b200 as j
    datas, headers = frame_sets(golden_dir)[name]
    frames = [j.ParsedFrame(d) for d in datas]
    tmaps = [transform_map(pf) for pf in frames]
    runs = []
    for ctx in contexts:
        outs = []
        for fmt in (XYB, U8):
            b, o = decode(ctx, frames, fmt)
            for i, tm in enumerate(tmaps):
                check_plan(b, i, tm, f"{name} frame {i}")
            b.close()
            outs += o
        runs.append(outs)
    for i, (a, b) in enumerate(zip(*runs)):
        assert np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8)), \
            f"{name}: output {i} differs between the one-SM and the full schedule"
    if headers is None:
        return
    b, _ = decode(contexts[1], frames, XYB, debug_stop=2)
    planes = [b.read_xyb(i, 0) for i in range(len(frames))]
    coeffs = [b.read_coeffs(i) for i in range(len(frames))]
    b.close()
    for i, pf in enumerate(frames):
        fr = fp.Frame(pf.desc(abi.FORMAT_RGB_F32)[0], header=headers[i])
        a, ma = fp.stage_a(fr, coeffs[i])
        fp.check("A", planes[i], a, ma, f"{name} frame {i}")


def test_partition_reaches_every_case(contexts, golden_dir):
    """The sets above reach: every class non-empty somewhere, empty classes, a group with only CTA-class varblocks."""
    import jxl_rs_b200 as j
    seen_class, empty_class, big_only = set(), set(), False
    for name, (datas, _) in frame_sets(golden_dir).items():
        for d in datas:
            for p in restated_plan(transform_map(j.ParsedFrame(d))):
                if p is None:
                    continue
                n = p[0]
                seen_class |= {c for c in range(5) if n[c]}
                empty_class |= {c for c in range(5) if not n[c]}
                big_only |= n[4] > 0 and sum(n[:4]) == 0
    assert seen_class == set(range(5)) and empty_class == set(range(5)) and big_only, (seen_class, empty_class, big_only)


def test_failed_plan_has_empty_classes(contexts):
    """Overlapping DCT32X32 varblocks overflow every group's coefficient area: the block plan fails, the batch reports
    JXG_ERR_INVALID_TRANSFORM, and every class of every group is empty; the unmutated twin is partitioned as restated."""
    import torch
    import jxl_rs_b200 as j
    import synth
    from tests.test_gpu_pipeline import overlapping_varblocks
    w, h = 300, 200
    fr = j.ParsedFrame(synth.encode_synthetic(w, h, 9, 0.5, 2, 1, 1))
    out = torch.empty((h, w, 3), dtype=torch.uint8, device="cuda:0")
    for mutate in (None, overlapping_varblocks):
        d, hf, off, ln, n = fr.desc(U8)
        keep = mutate(d, w, h) if mutate else None  # noqa: F841 - keeps the replacement buffers alive
        b = j.Batch(contexts[1], 1)
        try:
            b.add_desc(d, hf, off, ln, n, out.data_ptr(), w * 3, True)
            b.run()
            if mutate is None:
                b.wait()
                tm = transform_map(fr)
            else:
                with pytest.raises(abi.JxgError) as e:
                    b.wait()
                assert e.value.code == -8, e.value  # JXG_ERR_INVALID_TRANSFORM
                import ctypes as C
                xb, yb = (w + 7) // 8, (h + 7) // 8
                tm = np.frombuffer(C.string_at(d.transform_map, xb * yb), np.uint8).reshape(yb, xb)
            plans = check_plan(b, 0, tm, f"mutated={mutate is not None}")
            assert all(p is None for p in plans) if mutate else all(p is not None for p in plans)
        finally:
            b.close()
