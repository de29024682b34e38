"""XYB-encoded (lossy) Modular frames on the host: the parse accepts them with their LfQuantFactors and three coded
colour channels (also for a grey colour encoding), refuses those with Gaborish or EPF, keeps every other refusal, and
the CPU checker's Y, X, B channels of the fixture and of synthetic frames agree with the front-end's plan and with
the synthetic writer's source channels. tests/golden/jxl/bicycles.jxl is a byte-identical copy of the reference's
conformance image of that name (1024x631, XYB Modular, custom LfQuantFactors, global Squeeze, Gaborish and EPF off)."""
import json
import os

import numpy as np
import pytest

import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from tests import oracle_binding as ob

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "jxl")
UNSUPPORTED, OUT_OF_BOUNDS, ARGUMENT, INVALID_OUTPUT = -2, -3, -22, -9  # JXG_ERR_*
DEFAULT_QUANT = (1 / 4096, 1 / 512, 1 / 256)
CUSTOM_F16 = (0.0625, 0.25, 0.5)  # the factors times 128, as written: 1/2048, 1/512, 1/256


def bicycles():
    return open(os.path.join(GOLDEN, "bicycles.jxl"), "rb").read()


def features(data):
    import ctypes as C
    lib = ob._load_modular()
    lib.jxo_modular_features.restype = C.c_int64
    buf = C.create_string_buffer(1 << 16)
    n = lib.jxo_modular_features(data, len(data), buf, len(buf))
    assert n > 0
    return json.loads(buf.value.decode())


def test_bicycles_parses_as_an_xyb_frame():
    data = bicycles()
    fr = j.ModularParsedFrame(data)
    assert (fr.width, fr.height, fr.info.encoding, fr.info.num_groups) == (1024, 631, 1, 12)
    c = fr.colour(abi.FORMAT_RGB_U8)
    assert c["xyb"] and c["colour_channels"] == 3
    # the file's own LfQuantFactors (f16 values / 128), not the defaults
    assert np.allclose(c["lf_quant"], (2 ** -15, 2 ** -11, 2 ** -11), rtol=0, atol=0)
    f = features(data)
    assert f["global_transforms"] == ["squeeze(16 steps)"] and f["groups"] == 12
    # the inverse plan: 49 coded channels, then one buffer per unsqueeze of a channel (23 horizontal, 23 vertical)
    assert len(fr.region_plan((0, 0, fr.width, fr.height))[1]) == 49 + 46


@pytest.mark.parametrize("squeeze", [0, 1])
@pytest.mark.parametrize("q", [None, CUSTOM_F16])
def test_synthetic_factors_and_channels(squeeze, q):
    data = synth.encode_modular(333, 277, 9, rct=0, squeeze=squeeze, xyb={"lf_quant": q})
    c = j.ModularParsedFrame(data).colour()
    want = DEFAULT_QUANT if q is None else tuple(v / 128 for v in q)
    assert c["xyb"] and c["colour_channels"] == 3
    assert np.array_equal(np.float32(c["lf_quant"]), np.float32(want))
    _, planes = ob.decode_modular_file(data, planes=True)
    assert np.array_equal(planes, synth.modular_xyb_source(333, 277, 9, q))


def test_grey_xyb_codes_three_channels():
    grey_xyb = j.ModularParsedFrame(synth.encode_modular(200, 120, 3, rct=0, xyb={"colour": 6}))
    assert grey_xyb.colour()["colour_channels"] == 3
    d = grey_xyb.colour()["desc"]
    m = np.array(list(d.opsin_inverse_matrix)).reshape(3, 3)
    assert np.allclose(m[0], m[1]) and np.allclose(m[1], m[2])  # grey: the luminance row in every output channel
    lossless_grey = j.ModularParsedFrame(open(os.path.join(GOLDEN, "grayscale_public_university.jxl"), "rb").read())
    c = lossless_grey.colour()
    assert not c["xyb"] and c["colour_channels"] == 1 and c["lf_quant"] is None


def test_output_colour_matches_the_vardct_path():
    """The output stage of an XYB Modular frame is the one a VarDCT frame with the same image header gets."""
    for kw in ({"colour": c} for c in range(8)):
        m = j.ModularParsedFrame(synth.encode_modular(64, 40, 5, rct=0, xyb=kw)).colour(abi.FORMAT_RGB_F16)["desc"]
        v = j.ParsedFrame(synth.encode_synthetic(64, 40, 5, **kw)).desc(abi.FORMAT_RGB_F16)[0]
        for name in ("output_tf", "output_gamma", "intensity_target", "orientation", "output_format"):
            assert getattr(m, name) == getattr(v, name), (kw, name)
        for name in ("opsin_biases", "output_luminances", "opsin_inverse_matrix"):
            assert list(getattr(m, name)) == list(getattr(v, name)), (kw, name)


@pytest.mark.parametrize("kw", [{"gab": 1}, {"epf_iters": 1}, {"epf_iters": 3}, {"gab": 1, "epf_iters": 2}])
def test_filters_are_refused(kw):
    with pytest.raises(abi.JxgError) as e:
        j.ModularParsedFrame(synth.encode_modular(300, 200, 4, rct=0, xyb=kw))
    assert e.value.code == UNSUPPORTED and "Gaborish or EPF" in str(e.value)
    j.ModularParsedFrame(synth.encode_modular(300, 200, 4, rct=0, xyb={}))  # the twin without filters


def test_other_refusals_still_hold_on_xyb_files():
    data = synth.encode_modular(600, 520, 4, rct=0, squeeze=1, xyb={})
    with pytest.raises(abi.JxgError) as e:  # a cut file
        j.ModularParsedFrame(data[:len(data) - 100])
    assert e.value.code == OUT_OF_BOUNDS
    with pytest.raises(abi.JxgError) as e:  # a VarDCT frame
        j.ModularParsedFrame(synth.encode_synthetic(64, 64, 1))
    assert e.value.code == UNSUPPORTED
    for name in ("noise.jxl", "progressive_ac.jxl"):  # XYB files the Modular path refuses
        with pytest.raises(abi.JxgError) as e:
            j.ModularParsedFrame(open(os.path.join(GOLDEN, name), "rb").read())
        assert e.value.code == UNSUPPORTED


def test_region_plan_of_an_xyb_frame():
    """The cone of an XYB frame is the cone of its integer plan: the conversion is per pixel."""
    fr = j.ModularParsedFrame(bicycles())
    groups, arena, need = fr.region_plan((0, 0, fr.width, fr.height))
    assert groups == list(range(12))
    _, planes = ob.decode_modular_file(bicycles(), planes=True)
    assert planes.shape == (3, 631, 1024)
    groups, _, _ = fr.region_plan((1000, 600, 24, 31))
    assert 0 < len(groups) <= 12
