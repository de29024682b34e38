"""The device VarDCT AC coefficient decode (Batch.read_coeffs) against tests/vardct_ref.py on the token-level frames of
test_vardct_ref.py, bit for bit, with the entropy kernel instance of every frame asserted through
Batch.entropy_stats(): k_entropy_lean with and without the (4, 2, 0) form and the shared-memory context map, at 4 and
8 lanes per warp, k_entropy_fast and k_entropy. Mixed batches, the decode errors through the stream status and the
coefficient-entry width refusal are checked too."""
import numpy as np
import pytest

from jxl_rs_b200 import abi
from tests import test_vardct_ref as T
from tests import vardct_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import jxl_rs_b200 as j
    c = j.JxgContext(0)
    yield c
    c.close()


def gpu_decode(ctx, files):
    """Coefficients of every frame and the batch's entropy route."""
    import torch
    import jxl_rs_b200 as j
    frames = [j.ParsedFrame(f) for f in files]
    outs = [torch.empty((fr.height, fr.width, 3), dtype=torch.uint8).pin_memory() for fr in frames]
    b = j.Batch(ctx, len(frames))
    try:
        for fr, o in zip(frames, outs):
            b.add(fr, o.data_ptr(), fr.width * 3, abi.FORMAT_RGB_U8, False)
        b.run()
        route = b.entropy_stats()
        b.wait()
        return [b.read_coeffs(i) for i in range(len(frames))], route
    finally:
        b.close()


# expected route of each frame alone: kernel, and for the lean kernel its (4, 2, 0) and shared-memory forms
ROUTES = {
    "default_420": ("lean", True, True), "one_block_context": ("lean", False, True), "lf_x": ("lean", False, True),
    "lf_y": ("lean", False, True), "lf_b": ("lean", False, True), "lf_all64": ("lean", False, True),
    "qf15": ("lean", True, True), "hist3": ("lean", True, False), "hist_groups": ("lean", True, False),
    "shapes_large": ("lean", True, True), "thin": ("lean", True, True), "flat": ("lean", True, True),
    "ragged_tall_wide": ("lean", True, True), "entry_edges": ("lean", False, True),
    "prefix": ("fast", None, None), "orders": ("slow", None, None), "passes11": ("slow", None, None),
    "passes2_wrap": ("slow", None, None), "lz77": ("slow", None, None),
}


def _check_route(route, kernel, a420, smem, n):
    assert route[kernel] == n and sum(route[k] for k in ("lean", "fast", "slow")) == n, route
    if kernel == "lean":
        assert route["lean_all_420"] == a420 and route["lean_ctx_smem"] == smem and route["lean_S"] == 4, route


@pytest.mark.parametrize("name", T.CASES)
def test_device_equals_model(ctx, name):
    f, data = T.model(name)
    (coeffs,), route = gpu_decode(ctx, [data])
    _check_route(route, *ROUTES[name], f.num_groups)
    assert np.array_equal(coeffs, f.coeffs), name


def test_mixed_batches(ctx):
    """A (4, 2, 0) frame beside a frame with other configurations decodes on the general lean form; a frame whose
    context map does not fit the 16 KB staging area moves the whole batch to the global-memory form; ANS, prefix and
    multi-pass frames decode together."""
    for names, a420, smem in ((["default_420", "lf_all64", "qf15"], False, True),
                              (["hist3", "default_420", "thin"], True, False),
                              (["default_420", "prefix", "passes2_wrap", "lz77", "flat"], True, True)):
        models = [T.model(n) for n in names]
        coeffs, route = gpu_decode(ctx, [d for _, d in models])
        assert route["lean_all_420"] == a420 and route["lean_ctx_smem"] == smem, (names, route)
        for (f, _), c in zip(models, coeffs):
            assert np.array_equal(c, f.coeffs)


def test_eight_lanes_per_warp():
    """With three live contexts and at least 2048 lean streams the lean kernel runs 8 lanes per warp: one 4096 x 4096
    model frame (256 groups) added eight times."""
    import synth
    import jxl_rs_b200 as j
    rng = np.random.default_rng(4096)
    xb = yb = 512
    f = R.Frame(4096, 4096, T.tile(xb, yb, rng, [5, 5, 4, 0]), T.lf_field(rng, xb, yb), R.BlockContextMap(), 1,
                [T.one_pass(clusters=4)], [0] * 256)
    f.decode(T.chooser(4096, cap=24))
    data = synth.encode_vardct_tokens(f.spec)
    ctxs = [j.JxgContext(0) for _ in range(3)]
    try:
        coeffs, route = gpu_decode(ctxs[0], [data] * 8)
    finally:
        for c in ctxs:
            c.close()
    assert route["lean"] == 2048 and route["lean_S"] == 8, route
    for c in coeffs:
        assert np.array_equal(c, f.coeffs)


@pytest.mark.parametrize("case", ["invalid_num_nonzeros", "residual_nonzeros", "histogram_index"])
def test_refusal_with_twin_on_device(ctx, case):
    import synth
    bad, good, kind = T.refusal_pairs()[case]
    good, bad = good(), bad()
    (coeffs,), _ = gpu_decode(ctx, [synth.encode_vardct_tokens(good.spec)])
    assert np.array_equal(coeffs, good.coeffs)
    code = {"InvalidNumNonZeros": -5, "EndOfBlockResidualNonZeros": -6, "InvalidHistogramIndex": -4}[kind]
    with pytest.raises(abi.JxgError) as e:
        gpu_decode(ctx, [synth.encode_vardct_tokens(bad.spec)])
    assert e.value.code == code


@pytest.mark.parametrize("n", [6, 16])
@pytest.mark.parametrize("end", ["lo", "hi"])
def test_entry_width_refusal(ctx, n, end):
    """A coefficient entry holds [-2^(31-n), 2^(31-n) - 1] for 2^n coefficients per channel: the ends decode (the
    entry_edges frame), one past either end is refused with JXG_ERR_UNSUPPORTED, and the CPU oracle decodes it."""
    import synth
    rng = np.random.default_rng(n)
    t = 0 if n == 6 else 24
    size = 8 if n == 6 else 256
    lim = 1 << (31 - n)
    past = -lim - 1 if end == "lo" else lim

    def choose(ev):
        return 1, [past]
    f = R.Frame(size, size, [[0, 0, t, 5]], T.lf_field(rng, size // 8, size // 8), R.BlockContextMap(), 1,
                [T.one_pass(cfgs=[(4, 2, 0), (0, 0, 0)], log_alpha=8)], [0])
    f.decode(choose)
    data = synth.encode_vardct_tokens(f.spec)
    assert np.array_equal(T.oracle_coeffs(data), f.coeffs)
    with pytest.raises(abi.JxgError) as e:
        gpu_decode(ctx, [data])
    assert e.value.code == -2
