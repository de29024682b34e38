"""Squeeze on the device Modular path (ModularBatch) against tests/modular_ref.py, on the token-level frames of
test_modular_squeeze.py: planes and u8 bit-identical to the model at 1, 2 and 4 lanes per warp; a group-local Squeeze
is refused with JXG_ERR_UNSUPPORTED and the Squeeze refusals raise; one batch of frames of different sizes with the same
step structure (k_unsqueeze_h/v launches whose jobs have different shapes); frames whose step lists are prefixes of
each other, added in either order; and a frame refused by jxg_modular_batch_add leaves nothing in the batch."""
import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import modular_ref as M
from tests import test_gpu_modular_ref as G
from tests.gpu_modular import gpu_decode
from tests import test_modular_squeeze as S

pytestmark = pytest.mark.gpu

ctx = G.ctx
DEVICE_CASES = [n for n in S.CASES if n != "local_squeeze"]


def _check(frame, out, planes):
    assert np.array_equal(np.asarray(planes).reshape(-1), S.T.model_planes(frame).reshape(-1).astype(np.int32))
    assert np.array_equal(out, frame.u8)


@pytest.mark.parametrize("name", DEVICE_CASES)
def test_device_equals_model(ctx, name):
    frame, data = S.model(name)
    for lanes in (1, 2, 4):
        (out,), (planes,) = gpu_decode(ctx, [data], lanes)
        _check(frame, out, planes)


def test_local_squeeze_is_unsupported(ctx):
    _, data = S.model("local_squeeze")
    with pytest.raises(abi.JxgError) as e:
        gpu_decode(ctx, [data])
    assert e.value.code == -2, e.value  # JXG_ERR_UNSUPPORTED


@pytest.mark.parametrize("name,size,bad,good", S.REFUSALS, ids=[r[0] for r in S.REFUSALS])
def test_squeeze_refusals_on_device(ctx, name, size, bad, good):
    import synth
    G._refused_on_device(ctx, synth.encode_modular_tokens(S.refusal_frame(size, bad, False).spec))
    f = S.refusal_frame(size, good, True)
    (out,), (planes,) = gpu_decode(ctx, [synth.encode_modular_tokens(f.spec)])
    _check(f, out, planes)


STEPS = [(True, False, 1, 2), (False, True, 0, 3), (True, True, 0, 3), (False, False, 2, 1)]


def _steps_frame(w, h, steps, seed, lz=None):
    import synth
    rng = np.random.default_rng(seed)
    f = M.Frame(w, h, M.random_tree(rng, 4, S.PROPS), group_shift=0, transforms=[("squeeze", list(steps))])
    f.decode(M.picture_chooser(seed, p_small=0.3, p_huge=0.02))
    spec = f.spec
    if lz is not None:
        from tests import test_modular_lz77 as L
        spec = dict(spec, lz77=dict(L.ERROR_LZ, mode=2, multipliers=f.stream_widths, fault=lz.get("fault")))
    return f, synth.encode_modular_tokens(spec)


def test_batch_of_different_sizes(ctx):
    """One step structure on frames of 9 x 5 up to 300 x 150: each k_unsqueeze_h/v launch carries jobs of different
    shapes, and the threads past a small job's rows or columns exit early."""
    frames = [_steps_frame(w, h, STEPS, 40 + i) for i, (w, h) in enumerate([(300, 150), (9, 5), (64, 64), (131, 20),
                                                                            (50, 37)])]
    for lanes in (1, 4):
        outs, planes = gpu_decode(ctx, [d for _, d in frames], lanes)
        for (f, _), o, p in zip(frames, outs, planes):
            _check(f, o, p)


def test_step_lists_that_are_prefixes_in_either_order(ctx):
    """A frame whose undo plan is a prefix of another's shares the first levels; the order of adding must not
    matter."""
    short = _steps_frame(70, 50, STEPS[2:], 50)  # its plan is the first four levels of the long one's
    long_ = _steps_frame(80, 40, STEPS, 51)
    for pair in ((short, long_), (long_, short)):
        outs, planes = gpu_decode(ctx, [d for _, d in pair], 2)
        for (f, _), o, p in zip(pair, outs, planes):
            _check(f, o, p)


def test_refused_frame_leaves_the_batch_unchanged(ctx):
    """A and C share one step structure, B (its Squeeze undone in another order, and an LZ77 stream that starts with a
    copy) is refused at the structure check after its streams were staged. wait() reports no error, A and C equal the
    model, lz77_stats counts A and C only, in either order of A and C."""
    a = _steps_frame(140, 60, STEPS, 60, lz={})
    c = _steps_frame(96, 70, STEPS, 61, lz={})
    b = _steps_frame(140, 60, [(False, True, 0, 3), (True, True, 0, 3)], 62, lz={"fault": (1, 2)})
    _, alone, alone_stats = gpu_decode(ctx, [a[1], c[1]], 2, lz77_stats=True)
    assert alone_stats["lz77_streams"] > 0
    for first, last in ((a, c), (c, a)):
        outs, planes, stats = gpu_decode(ctx, [first[1], b[1], last[1]], 2, lz77_stats=True, refused=(1,))
        assert stats == alone_stats, (stats, alone_stats)
        for (f, _), o, p in zip((first, last), outs, planes):
            _check(f, o, p)
