"""The device's table walk (m_channel_lut in modular_kernels.cu) against tests/modular_ref.py on the frames of
test_modular_walk_table.py: i32 planes and u8 pixels bit-identical to the model at 1, 2 and 4 lanes per warp, with
ModularBatch.walk_stats() counting the routes the frames were designed for; the LZ77 forms of two cases; all frames in
one batch; and a table-walk frame beside its generic-walk twin."""
import numpy as np
import pytest

from tests import test_modular_walk_table as W
from tests.gpu_modular import gpu_decode
from tests.test_modular_ref import model_planes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


def _check(it, out, planes):
    assert np.array_equal(np.asarray(planes).reshape(-1), model_planes(it.frame).reshape(-1).astype(np.int32)), it.label
    assert np.array_equal(out, it.frame.u8), it.label


@pytest.mark.parametrize("name", W.CASES)
def test_device_equals_model(ctx, name):
    for it, data in W.items(name):
        for lanes in (1, 2, 4):
            (out,), (planes,), walks = gpu_decode(ctx, [data], lanes, walk_stats=True)
            _check(it, out, planes)
            assert walks == W.expected_walk_stats([it]), (it.label, walks)


@pytest.mark.parametrize("name", sorted(W.LZ77_CASES))
def test_lz77_device_equals_model(ctx, name):
    """The LZ = true instances: every group stream of the frame uses LZ77 and takes the table walk it was designed for."""
    for it, data, census in W.lz77_items(name):
        assert census["copies"] > 100
        for lanes in (1, 2, 4):
            (out,), (planes,), lz, walks = gpu_decode(ctx, [data], lanes, lz77_stats=True, walk_stats=True)
            _check(it, out, planes)
            assert lz["lz77_streams"] == len({g for g, _ in it.routes}), lz
            assert walks == W.expected_walk_stats([it]), (it.label, walks)


def test_mixed_batch(ctx):
    """Every frame of every case, and the LZ77 forms, in one batch (LZ77 streams in their own launch)."""
    its, files = [], []
    for name in W.CASES:
        for it, data in W.items(name):
            its.append(it)
            files.append(data)
    for name in sorted(W.LZ77_CASES):
        for it, data, _ in W.lz77_items(name):
            its.append(it)
            files.append(data)
    outs, planes, walks = gpu_decode(ctx, files, 2, walk_stats=True)
    for it, o, p in zip(its, outs, planes):
        _check(it, o, p)
    assert walks == W.expected_walk_stats(its), walks


def test_table_frame_beside_its_generic_twin(ctx):
    """The clamp-edge frame whose splits sit at the table's ends and its twin whose splits sit one beyond them, in one
    batch in both orders: the first takes the table walk, the second the generic one, and both decode as the model."""
    pair = W.items("clamp_edges")
    for order in (pair, pair[::-1]):
        for lanes in (1, 4):
            outs, planes, walks = gpu_decode(ctx, [d for _, d in order], lanes, walk_stats=True)
            for (it, _), o, p in zip(order, outs, planes):
                _check(it, o, p)
            assert walks == {"generic": 12, "single_leaf": 0, "by_property": {5: 4, 6: 4, 7: 4}, "table_wp": 0}, walks
