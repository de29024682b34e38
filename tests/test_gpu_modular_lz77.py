"""LZ77 group streams on the device Modular path (ModularBatch): the frames of test_modular_lz77.py at 1, 2 and 4 lanes
per warp, bit-exact against the CPU oracle and the token-level model; the LZ77 streams take their own launch
(lz77_stats), a batch mixes frames with and without copies, the two LZ77 errors come back from wait() as JXG_ERR_LZ77
for the right frame and group while the other frame decodes, and a 4096^2 run-length frame decodes to its source."""
import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import test_modular_lz77 as L
from tests.gpu_modular import gpu_decode

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


@pytest.mark.parametrize("lz", [1, 2])
@pytest.mark.parametrize("kw", [dict(rct=6, squeeze=0, tree_kind=1), dict(rct=6, squeeze=1, tree_kind=2),
                                dict(rct=0, squeeze=0, tree_kind=0), dict(rct=6, squeeze=0, tree_kind=3)],
                         ids=["rct_tree", "squeeze_wp", "gradient", "ref_props"])
def test_writer_frames_equal_the_oracle(ctx, kw, lz):
    import synth
    w, h = 600, 520
    src = L.flat_picture(w, h)
    data = synth.encode_modular(w, h, 7, source=src, lz77=lz, **kw)
    ref_out, ref_planes = L.oracle(data)
    for lanes in (1, 2, 4):
        (out,), (planes,), st = gpu_decode(ctx, [data], lanes, lz77_stats=True)
        assert np.array_equal(planes, ref_planes) and np.array_equal(out, ref_out) and np.array_equal(out, src)
        assert st["lz77_streams"] == 9 and st["rle_streams"] == (9 if lz == 1 else 0), st
        assert st["window_bytes"] > 0


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", L.TOKEN_CASES)
def test_token_frames_equal_the_model(ctx, name, mode):
    frame, data, _ = L.token_frame(name, mode)
    for lanes in (1, 2, 4):
        (out,), (planes,), st = gpu_decode(ctx, [data], lanes, lz77_stats=True)
        assert np.array_equal(np.asarray(planes).reshape(-1), L.model_planes(frame).reshape(-1).astype(np.int32))
        assert np.array_equal(out, frame.u8)
        assert st["lz77_streams"] > 0


def test_copy_at_distance_two_to_the_twenty(ctx):
    planes, data, _ = L.long_stream_frame()
    for lanes in (1, 4):
        _, (got,), st = gpu_decode(ctx, [data], lanes, lz77_stats=True)
        assert np.array_equal(got, planes.astype(np.int32))
        assert st["lz77_streams"] == 2 and st["window_bytes"] == 2 * 4 << 20


def test_mixed_batch(ctx):
    """Run-length, general and copy-free frames in one batch (frames of one batch share their global transforms); the
    copy-free frame decodes as it does alone."""
    import synth
    w, h = 600, 520
    src = L.flat_picture(w, h, 1)
    files = [synth.encode_modular(w, h, 7, source=src, lz77=1), synth.encode_modular(w, h, 7, source=src, lz77=0),
             synth.encode_modular(w, h, 7, source=src, tree_kind=2, lz77=2)]
    for lanes in (1, 2, 4):
        outs, planes, st = gpu_decode(ctx, files, lanes, lz77_stats=True)
        assert st["lz77_streams"] == 18 and st["rle_streams"] == 9, st
        for o in outs:
            assert np.array_equal(o, src)
        (alone_out,), (alone_planes,), st0 = gpu_decode(ctx, files[1:2], lanes, lz77_stats=True)
        assert st0["lz77_streams"] == 0
        assert np.array_equal(alone_planes, planes[1]) and np.array_equal(alone_out, outs[1])


@pytest.mark.parametrize("fault", [1, 2], ids=["copy_first", "length_overflow"])
def test_lz77_errors_are_reported(ctx, fault):
    """Section 4 of the frame is HF group 2 (one global section, one LF group before it)."""
    good_frame, good, _ = L.token_frame("ans_tree", 2, lz=L.ERROR_LZ)
    _, bad, _ = L.token_frame("ans_tree", 2, fault=(fault, 4), lz=L.ERROR_LZ)
    for lanes in (1, 4):
        (out, _), (planes, _), err = gpu_decode(ctx, [good, bad], lanes, expect_error=True)
        assert err is not None and err.code == -10 and "frame 1 group 2" in str(err), err
        assert np.array_equal(np.asarray(planes).reshape(-1), L.model_planes(good_frame).reshape(-1).astype(np.int32))
        assert np.array_equal(out, good_frame.u8)


def test_large_run_length_frame(ctx):
    import synth
    w = h = 4096
    src = L.flat_picture(w, h, 2)
    data = synth.encode_modular(w, h, 1, source=src, lz77=1)
    (out,), _, st = gpu_decode(ctx, [data], 4, lz77_stats=True)
    assert np.array_equal(out, src)
    assert st["lz77_streams"] == 256 and st["rle_streams"] == 256
