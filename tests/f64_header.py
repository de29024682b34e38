"""What the frame-level header fields a frame was written with decode to, restated from the reference text (not a test
module). The fields are those of synth.encode_synthetic(header=...): every float an f16 bit pattern.

  RestorationFilter        frame_header.rs:146-234   Gaborish weights, EPF sharpness LUT, channel scales, sigma fields
  ColorCorrelationParams   color_correlation_map.rs:42-72   color_factor selector, base correlations, LF factors
  OpsinInverseMatrix       transform_data.rs:18-32   opsin inverse matrix, opsin biases, quant biases
  CfL tile maps            modular/mod.rs:1018-1030  each value clamped to i8

decode() gives the values as float64 (f16 -> f32 -> f64 is exact) or raises Refused where the reference refuses the
header: a non-finite f16 in a field that is read (encodings.rs:59-74 via the f16 coder, color_correlation_map.rs:55-57),
or a base correlation above 4 (color_correlation_map.rs:60-62; negative bases are accepted). f64_pipeline.Frame takes
these values, not the descriptor's, and asserts that the descriptor holds the same ones."""
import numpy as np

from tests.f64_quant import f16

# frame_header.rs:157-231, color_correlation_map.rs:29-38, transform_data.rs:24-31, as the reference's f32 literals
DEFAULTS = {
    "gab_w1": [0.115169525] * 3, "gab_w2": [0.061248592] * 3,
    "epf_sharp_lut": [0.0, 1 / 7, 2 / 7, 3 / 7, 4 / 7, 5 / 7, 6 / 7, 1.0],
    "epf_channel_scale": [40.0, 5.0, 3.5],
    "epf_quant_mul": 0.46, "epf_pass0_sigma_scale": 0.9, "epf_pass2_sigma_scale": 6.5, "epf_border_sad_mul": 2 / 3,
    "color_factor": 84, "base_x": 0.0, "base_b": 1.0,
    "opsin_inverse_matrix": [11.031566901960783, -9.866943921568629, -0.16462299647058826,
                             -3.254147380392157, 4.418770392156863, -0.16462299647058826,
                             -3.6588512862745097, 2.7129230470588235, 1.9459282392156863],
    "opsin_biases": [-0.0037930732552754493] * 3,
    "quant_biases": [0.0, 0.0, 0.0, 0.145],
}
DEFAULTS = {k: np.float32(v).astype(np.float64) if not isinstance(v, int) else v for k, v in DEFAULTS.items()}
# 1.0 - x of the quant biases is an f32 subtraction in the reference's literal
DEFAULTS["quant_biases"][:3] = (np.float32(1.0) - np.float32([0.05465007330715401, 0.07005449891748593,
                                                              0.049935103337343655])).astype(np.float64)

# The fields of the descriptor (include/jxg.h JxgFrameDesc) each key is compared with
DESC_FIELD = {"gab_w1": "gab_w1", "gab_w2": "gab_w2", "epf_sharp_lut": "epf_sharp_lut",
              "epf_channel_scale": "epf_channel_scale", "epf_quant_mul": "epf_quant_mul",
              "epf_pass0_sigma_scale": "epf_pass0_sigma_scale", "epf_pass2_sigma_scale": "epf_pass2_sigma_scale",
              "epf_border_sad_mul": "epf_border_sad_mul", "color_factor": "color_factor",
              "base_x": "base_correlation_x", "base_b": "base_correlation_b",
              "opsin_biases": "opsin_biases", "quant_biases": "quant_biases"}
# The descriptor's opsin_inverse_matrix is the written one re-targeted to the output colour encoding (include/jxg.h;
# the colour derivation is restated in test_kat_colour.py): it equals the written matrix for sRGB-primaries output only.

# opsin_inverse.jxl's CustomTransformData (EPF 1, Gaborish on, other fields default), as f16 bit patterns
OPSIN_INVERSE_FIXTURE = {"opsin": {"matrix": [0x4a00, 0xc800, 0xae66, 0xc400, 0x4500, 0x0000, 0xc400, 0x4400, 0x4200],
                                   "biases": [0x9818, 0x9d1e, 0x9c18],
                                   "quant_biases": [0x4000, 0x3c00, 0x4200, 0x30a3]}}


class Refused(ValueError):
    """The reference refuses a frame with these header fields."""


def color_factor(sel, bits):
    """color_correlation_map.rs:46-51."""
    return {0: 84, 1: 256, 2: (bits & 0xFF) + 2, 3: (bits & 0xFFFF) + 258}[sel & 3]


def _finite(bits, what):
    v = f16(np.asarray(bits, np.uint16))
    if not np.all(np.isfinite(v)):
        raise Refused(f"non-finite f16 in {what}")
    return v


def decode(header, gab=1, epf_iters=2):
    """The float64 value of every field (DEFAULTS' keys) a frame written with `header` (synth.encode_synthetic's dict)
    carries, with Gaborish `gab` and `epf_iters`: the groups the reader skips (Gaborish off, EPF 0) keep their
    defaults whatever the dict holds. Raises Refused as the reference does."""
    out = {k: (np.array(v) if not np.isscalar(v) else v) for k, v in DEFAULTS.items()}
    header = header or {}
    if gab and "gab" in header:
        w = _finite(header["gab"], "Gaborish weights")
        out["gab_w1"], out["gab_w2"] = w[0::2].copy(), w[1::2].copy()
    if epf_iters > 0:
        if "sharp" in header:
            out["epf_sharp_lut"] = _finite(header["sharp"], "epf_sharp_lut")
        if "weight" in header:
            out["epf_channel_scale"] = _finite(header["weight"], "epf weights")[:3]
        if "sigma" in header:
            s = _finite(header["sigma"], "epf sigma")
            (out["epf_quant_mul"], out["epf_pass0_sigma_scale"], out["epf_pass2_sigma_scale"],
             out["epf_border_sad_mul"]) = (float(v) for v in s)
    if "color" in header:
        cc = header["color"]
        out["color_factor"] = color_factor(*cc.get("factor", (0, 0)))
        bx, bb = _finite([cc.get("base_x", 0), cc.get("base_b", 0x3C00)], "base correlations")
        if bx > 4.0 or bb > 4.0:
            raise Refused("base colour correlation above 4")
        out["base_x"], out["base_b"] = float(bx), float(bb)
    if "opsin" in header:
        op = header["opsin"]
        out["opsin_inverse_matrix"] = _finite(op["matrix"], "opsin matrix")
        out["opsin_biases"] = _finite(op["biases"], "opsin biases")
        out["quant_biases"] = _finite(op["quant_biases"], "quant biases")
    return out


def cfl_maps(header, ty, tx):
    """The CfL tile maps (ytox, ytob) the decoder holds, (ty, tx) int32 each: the written values clamped to i8;
    None when the header leaves them to the writer."""
    if not header or "cfl" not in header:
        return None
    return tuple(np.clip(np.asarray(m, np.int64).reshape(ty, tx), -128, 127).astype(np.int32) for m in header["cfl"])


def descriptor_values(d):
    """The descriptor's value of every DEFAULTS key, as float64 (color_factor as int)."""
    out = {}
    for k, f in DESC_FIELD.items():
        v = getattr(d, f)
        out[k] = int(v) if k == "color_factor" else (np.array(list(v), np.float64) if hasattr(v, "__len__") else float(v))
    return out


def differing(a, b):
    """Keys whose values differ between two value dicts (exact comparison)."""
    return [k for k in DESC_FIELD if not np.array_equal(np.asarray(a[k], np.float64), np.asarray(b[k], np.float64))]


def f16_bits(v):
    """The f16 bit pattern of a value that f16 holds exactly (asserted)."""
    h = np.float16(v)
    assert float(h) == float(v), f"{v} is not an f16 value"
    return int(np.array(h).view(np.uint16))
