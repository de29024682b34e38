"""The device Modular path (ModularBatch) against tests/modular_ref.py on the token-level frames of
test_modular_ref.py: i32 planes and u8 pixels bit-identical to the model at 1, 2 and 4 lanes per warp, a mixed batch,
and the tree, RCT and palette refusals, which must raise JxgError and never decode. The palette cases run the
device's palette look-up (k_modular_palette) on explicit, cube, beyond-cube and negative indices."""
import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import modular_ref as M
from tests import test_modular_ref as T
from tests.gpu_modular import gpu_decode

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


def _check(frame, out, planes):
    assert np.array_equal(np.asarray(planes).reshape(-1), T.model_planes(frame).reshape(-1).astype(np.int32))
    assert np.array_equal(out, frame.u8)


@pytest.mark.parametrize("name", T.CASES)
def test_device_equals_model(ctx, name):
    frame, data = T.model(name)
    for lanes in (1, 2, 4):
        (out,), (planes,) = gpu_decode(ctx, [data], lanes)
        _check(frame, out, planes)


def test_mixed_batch(ctx):
    """Frames of one geometry with different global trees, WeightedHeaders, local trees and local RCTs in one batch."""
    import synth
    rng = np.random.default_rng(77)
    frames = []
    for i in range(4):
        groups = {g: {"wp": T._wp(rng), "rct": [(0, int(rng.integers(0, 42)))],
                      "tree": M.random_tree(rng, 3, [0, 9, 15], leaf_preds=[6, 13, 4]) if (g + i) % 2 else None}
                  for g in range(4)}
        f = M.Frame(140, 130, M.random_tree(rng, 4, T.ALL_PROPS, wide_leaves=i == 3), group_shift=0, groups=groups,
                    global_wp=T._wp(rng) if i % 2 else None)
        frames.append(f.decode(M.picture_chooser(100 + i, p_huge=0.05 * i)))
    files = [synth.encode_modular_tokens(f.spec) for f in frames]
    outs, planes = gpu_decode(ctx, files, 2)
    for f, o, p in zip(frames, outs, planes):
        _check(f, o, p)


def _refused_on_device(ctx, data):
    with pytest.raises(abi.JxgError):
        gpu_decode(ctx, [data])


@pytest.mark.parametrize("name,bad,good", T.REFUSALS, ids=[r[0] for r in T.REFUSALS])
@pytest.mark.parametrize("where", ["global", "local"])
def test_tree_refusals_on_device(ctx, name, bad, good, where):
    import synth
    base = [("leaf", 5, 0, 0, 0)]
    for tree, ok in ((bad, False), (good, True)):
        f = T._refusal_frame(tree, ok) if where == "global" else T._refusal_frame(base, ok, groups={0: {"tree": tree}})
        data = synth.encode_modular_tokens(f.spec)
        if ok:
            (out,), (planes,) = gpu_decode(ctx, [data])
            _check(f, out, planes)
        else:
            _refused_on_device(ctx, data)


@pytest.mark.parametrize("rct,grey,local", [((0, 42), False, False), ((0, 42), False, True), ((1, 6), False, False),
                                            ((1, 6), False, True), ((0, 6), True, False)])
def test_transform_refusals_on_device(ctx, rct, grey, local):
    import synth
    kw = {"groups": {2: {"rct": [rct]}}} if local else {"global_rct": [rct]}
    f = T._refusal_frame([("leaf", 5, 0, 0, 0)], False, grey=grey, **kw)
    _refused_on_device(ctx, synth.encode_modular_tokens(f.spec))


@pytest.mark.parametrize("name,kw", T.PALETTE_REFUSALS, ids=[r[0] for r in T.PALETTE_REFUSALS])
def test_palette_range_refusals_on_device(ctx, name, kw):
    import synth
    f = T._refusal_frame([("leaf", 5, 0, 0, 0)], False, **kw)
    _refused_on_device(ctx, synth.encode_modular_tokens(f.spec))
