"""The host side of the 1:8 thumbnail path (jxg_lf_parse_file), no device needed: it accepts and refuses what
jxg_parse_file does with the same JxgImageInfo, reads nothing behind the last LF-group section, and the float64
expectation the GPU tests compare thumbnails with has the thumbnail's display shape."""
import ctypes as C
import glob
import os
import random
import types

import numpy as np
import pytest

import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from tests import f64_pipeline as fp

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "jxl", "*.jxl")))
INFO_FIELDS = ("width", "height", "num_groups", "num_passes", "encoding", "hf_bytes", "coded_width", "coded_height",
               "orientation")


def synthetic_frames():
    """Synthetic VarDCT frames: several LF groups, sizes that are not multiples of 8 or 2048, every orientation,
    extra_precision 0..3, smoothing on and off, an LF chroma-from-luma that differs from the HF one, and LF streams
    coded with prefix codes and with LZ77 copies over ANS and over prefix codes (lf-e1 .. lf-e3)."""
    out = [("4100x2200", synth.encode_synthetic(4100, 2200, 11, profile=0)),
           ("2100x300", synth.encode_synthetic(2100, 300, 12, lf_tree=1)),
           ("257x129", synth.encode_synthetic(257, 129, 13)), ("7x5", synth.encode_synthetic(7, 5, 14))]
    out += [(f"o{o}", synth.encode_synthetic(300, 180, 20 + o, orientation=o)) for o in range(1, 9)]
    out += [(f"ep{ep}-skip{sk}", synth.encode_synthetic(2060, 530, 30 + ep, profile=0, lf_extra_precision=ep,
                                                        skip_lf_smoothing=bool(sk)))
            for ep in range(4) for sk in (0, 1)]
    out += [("lf-cfl", synth.encode_synthetic(2060, 530, 40, profile=0, lf_extra_precision=1,
                                              header={"color": {"ytox_lf": 37, "ytob_lf": -51}}))]
    out += lf_entropy_frames()
    return out


def lf_entropy_frames():
    """Frames with several LF groups whose LF streams use prefix codes (1), LZ77 copies over ANS (2) and over prefix
    codes (3), with the one-leaf and the weighted-predictor LF tree."""
    return [(f"lf-e{e}-t{t}", synth.encode_synthetic(2100, 600, 50 + e, profile=0, lf_tree=t, lf_entropy=e))
            for e in (1, 2, 3) for t in (0, 1)]


def parse(cls, data):
    try:
        return cls(data).info, 0
    except abi.JxgError as e:
        return None, e.code


def lf_code(data):
    return parse(j.LfParsedFrame, data)[1]


@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_same_answer_as_parse_file_on_fixtures(path):
    data = open(path, "rb").read()
    (full, c_full), (lf, c_lf) = parse(j.ParsedFrame, data), parse(j.LfParsedFrame, data)
    assert c_lf == c_full
    if c_full == 0:
        assert [getattr(lf, k) for k in INFO_FIELDS] == [getattr(full, k) for k in INFO_FIELDS]


def test_same_answer_as_parse_file_on_synthetic_frames():
    for name, data in synthetic_frames():
        (full, c_full), (lf, c_lf) = parse(j.ParsedFrame, data), parse(j.LfParsedFrame, data)
        assert c_full == 0 and c_lf == 0, name
        assert [getattr(lf, k) for k in INFO_FIELDS] == [getattr(full, k) for k in INFO_FIELDS], name


def test_lf_entropy_variants_code_the_same_lf_image():
    """The writer's LF entropy option changes only how the LF symbols are coded: the host's LF planes of each variant
    equal those of the ANS-coded frame with the same seed."""
    for e in (1, 2, 3):
        for t in (0, 1):
            ref, _ = lf_planes(synth.encode_synthetic(2100, 600, 50 + e, profile=0, lf_tree=t))
            got, _ = lf_planes(synth.encode_synthetic(2100, 600, 50 + e, profile=0, lf_tree=t, lf_entropy=e))
            assert got.view(np.uint32).tobytes() == ref.view(np.uint32).tobytes(), (e, t)


def test_modular_files_refused_alike():
    data = synth.encode_modular(300, 200, 3)
    assert parse(j.ParsedFrame, data)[1] == parse(j.LfParsedFrame, data)[1] == -2  # JXG_ERR_UNSUPPORTED


def lf_end(data):
    """The shortest prefix of a bare codestream the LF parse accepts (binary search; accepted prefixes are upward
    closed, checked by the callers)."""
    lo, hi = 1, len(data)
    while lo < hi:
        mid = (lo + hi) // 2
        if lf_code(data[:mid]) == 0:
            hi = mid
        else:
            lo = mid + 1
    return lo


@pytest.mark.parametrize("w,h", [(2100, 300), (4100, 2200)])
def test_reads_nothing_past_the_lf_groups(w, h):
    data = synth.encode_synthetic(w, h, 41, profile=0)
    info = j.ParsedFrame(data).info
    end = lf_end(data)
    # HfGlobal and the HF sections follow the last LF group: at least hf_bytes + 1 bytes are never needed
    assert end <= len(data) - info.hf_bytes - 1
    assert lf_code(data[:end - 1]) == -3  # JXG_ERR_OUT_OF_BOUNDS: cut inside the last LF-group section
    for cut in (end, end + 1, (end + len(data)) // 2, len(data) - 1):
        got = j.LfParsedFrame(data[:cut]).info
        assert [getattr(got, k) for k in INFO_FIELDS] == [getattr(info, k) for k in INFO_FIELDS]
    for cut in (end - 2, end - 100):
        assert lf_code(data[:cut]) == -3
    assert parse(j.ParsedFrame, data[:end])[1] == -3  # the whole-frame parse needs every section
    rng = random.Random(7)
    noisy = data[:end] + bytes(rng.randrange(256) for _ in range(len(data) - end))
    got = j.LfParsedFrame(noisy).info
    assert [getattr(got, k) for k in INFO_FIELDS] == [getattr(info, k) for k in INFO_FIELDS]


def test_single_section_frame_must_be_whole():
    data = synth.encode_synthetic(200, 120, 42)
    info = j.ParsedFrame(data).info
    assert info.num_groups == 1 and j.LfParsedFrame(data).info.hf_bytes == info.hf_bytes
    assert lf_code(data[:-1]) == -3


# ---------------------------------------------------------------------------------------------------------------------
# The float64 expectation of a thumbnail (used by tests/test_gpu_lf_thumbnail.py)
# ---------------------------------------------------------------------------------------------------------------------
def _arr(ptr, ctype, shape):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape=shape).copy()


def lf_planes(data):
    """The host front end's LF planes (jxg_parsed_desc lf[3]): X, Y, B float32 (yb, xb), and the descriptor."""
    d = j.ParsedFrame(data).desc(abi.FORMAT_RGB_F32)[0]
    xb, yb = (d.width + 7) // 8, (d.height + 7) // 8
    return np.stack([_arr(d.lf[c], C.c_float, (yb, xb)) for c in range(3)]), d


def expected_thumbnail(data, fmt):
    """(ref, mag, tf, orientation) for fp.check_output: f64_pipeline.stage_c of the LF planes under the output
    encoding jxg_parsed_desc gives for `fmt`; check_output applies the store and the orientation."""
    planes, _ = lf_planes(data)
    d = j.ParsedFrame(data).desc(fmt)[0]
    fr = types.SimpleNamespace(output_tf=int(d.output_tf), opsin_biases=np.array(list(d.opsin_biases), np.float64),
                               intensity_target=float(d.intensity_target), output_gamma=float(d.output_gamma),
                               output_luminances=np.array(list(d.output_luminances), np.float64),
                               opsin_inverse_matrix=np.array(list(d.opsin_inverse_matrix), np.float64).reshape(3, 3))
    ref, mag = fp.stage_c(fr, planes.astype(np.float64))
    return ref, mag, int(d.output_tf), int(d.orientation)


def test_expectation_shape_and_orientation():
    for name, data in synthetic_frames()[:12] + [(os.path.basename(p), open(p, "rb").read()) for p in GOLDEN]:
        if parse(j.ParsedFrame, data)[1]:
            continue
        lf = j.LfParsedFrame(data)
        ref, _, tf, o = expected_thumbnail(data, abi.FORMAT_RGB_U8)
        want = (-(-lf.info.height // 8), -(-lf.info.width // 8))
        assert (lf.height, lf.width) == want, name
        assert (lf.coded_height, lf.coded_width) == ref.shape[:2], name
        out = fp.orient(fp.store(fp.FMT_U8, ref, tf), o)
        assert out.shape[:2] == want, name
        if o >= 5:
            assert want == ref.shape[1::-1], name
