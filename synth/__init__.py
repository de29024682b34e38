"""Synthetic VarDCT .jxl generator (ctypes binding of synth/libjxlsynth.so). Test-data tooling."""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "libjxlsynth.so")
        if not os.path.exists(path):
            subprocess.check_call(["make", "-C", _HERE])
        _LIB = C.CDLL(path)
        _LIB.jxs_encode_synthetic.restype = C.c_int64
        _LIB.jxs_encode_synthetic.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.c_float, C.c_uint32, C.c_uint32,
                                              C.c_uint32, C.c_void_p, C.c_size_t]
        _LIB.jxs_encode_synthetic_ex.restype = C.c_int64
        _LIB.jxs_encode_synthetic_ex.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.c_float, C.c_uint32, C.c_uint32,
                                                 C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t,
                                                 C.c_void_p, C.c_size_t]
        _LIB.jxs_last_error.restype = C.c_char_p
        _LIB.jxs_set_threads.argtypes = [C.c_int]
        _LIB.jxs_encode_modular.restype = C.c_int64
        _LIB.jxs_encode_modular.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32,
                                            C.c_void_p, C.c_void_p, C.c_size_t]
        _LIB.jxs_modular_source.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p]
        _LIB.jxs_modular_source_ex.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p]
        _LIB.jxs_encode_modular_ex.restype = C.c_int64
        _LIB.jxs_encode_modular_ex.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                               C.c_void_p, C.c_void_p, C.c_size_t]
        _LIB.jxs_modular_last_error.restype = C.c_char_p
        _LIB.jxs_encode_modular_tokens.restype = C.c_int64
        _LIB.jxs_encode_modular_tokens.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    return _LIB


def encode_synthetic(width, height, seed, distance=1.0, epf_iters=2, gab=1, profile=1, lf_tree=0, entropy=0, orientation=1,
                     colour=0, dequant=None, x_qm_scale=3, b_qm_scale=2) -> bytes:
    """One synthetic VarDCT frame. profile 0: DCT8x8 only; 1: mixed transforms up to 32x32;
    2: also 64x64 / 64x32 / 32x64; 3: also the 128 / 256 families (DCT128X128 ... DCT256X256, transform types 21..26);
    4: profile 3 plus IDENTITY, DCT2X2 and AFV0-3 among the 8x8 blocks, so that every dequantisation table is used.
    Profile 4 gives those blocks random sparse coefficients instead of a forward transform: its frames are valid but
    do not reproduce the source picture, and the writer's PSNR round trip does not apply to them.
    lf_tree 0: LF image coded with one Gradient leaf per channel; 1: like libjxl (channel prefix, then a subtree on the
    weighted-predictor property with Weighted-predictor leaves). entropy 0: ANS-coded AC streams; 1: prefix codes; 2 / 3: the same with LZ77 copies.
    orientation: ImageMetadata.orientation 1..8. colour: embedded colour encoding (0 sRGB, 1 linear, 2 gamma 0.45455,
    3 P3 + PQ, 4 BT2100 + HLG, 5 custom primaries + DCI white + BT709, 6 grey, 7 E white + DCI curve).
    dequant: None (DequantMatrices all_default) or 17 entries, each None (library table) or a custom encoding in the
    form of tests/f64_quant.py (a dict with "mode" 1..7 and its parameters as f16 bit patterns), written as given,
    also when the decoder must refuse it. x_qm_scale, b_qm_scale: the frame header's 0..7. The coefficients are
    quantised with the tables the decoder computes from what is written."""
    profile = ((profile & 0xff) | ((lf_tree & 1) << 8) | ((entropy & 3) << 9) | (((orientation - 1) & 7) << 12)
               | ((colour & 15) << 16))
    lib = _lib()
    words = _dequant_words(dequant)
    arr = (C.c_uint32 * max(1, len(words)))(*[w & 0xFFFFFFFF for w in words])

    def run(buf, cap):
        if not words and (x_qm_scale, b_qm_scale) == (3, 2):
            return lib.jxs_encode_synthetic(width, height, seed, distance, epf_iters, gab, profile, buf, cap)
        return lib.jxs_encode_synthetic_ex(width, height, seed, distance, epf_iters, gab, profile, x_qm_scale, b_qm_scale,
                                           arr, len(words), buf, cap)
    cap = max(1 << 16, width * height * 2 + 4 * len(words))
    buf = C.create_string_buffer(cap)
    n = run(buf, cap)
    if n < 0:
        raise RuntimeError("synthetic encode failed: " + lib.jxs_last_error().decode())
    if n > cap:
        buf = C.create_string_buffer(n)
        n = run(buf, n)
    return buf.raw[:n]


def _dequant_words(dequant):
    """The flat u32 array of jxs_encode_synthetic_ex: per table the mode, then the (value, bits) fields in the order
    QuantEncoding::decode reads them (quant_weights.rs:117-255), then the RAW entries."""
    if dequant is None:
        return []
    assert len(dequant) == 17, "dequant takes one entry per table index"
    words = []
    for enc in dequant:
        if enc is None:
            words.append(0)
            continue
        mode = int(enc["mode"])
        fields = []

        def f16s(vals):
            fields.extend((int(v) & 0xFFFF, 16) for v in vals)

        def dct(p):  # DctQuantWeightParams::decode (quant_weights.rs:58-71): num_bands - 1, then 3 x num_bands
            fields.append((len(p[0]) - 1, 4))
            for row in p:
                f16s(row)
        if mode in (1, 2, 3, 4, 5):
            f16s(list(_flat(enc["w"])))
        if mode in (3, 4, 5, 6):
            dct(enc["dct"])
        if mode == 5:
            dct(enc["dct4"])
        if mode == 7:
            f16s([enc["den"]])
        words += [mode, len(fields)] + [x for fb in fields for x in fb]
        if mode == 7:
            import numpy as np
            words += np.asarray(enc["raw"], np.int64).ravel().tolist()
    return words


def _flat(v):
    for x in v:
        if hasattr(x, "__len__"):
            yield from _flat(x)
        else:
            yield x


def set_threads(n: int):
    """Worker threads inside each following encode_synthetic call (one large image); the bitstream does not depend
    on it. Batches of many frames keep 1 and encode frames in parallel instead."""
    _lib().jxs_set_threads(int(n))


def modular_source(width, height, seed, palette=0):
    """The 8-bit RGB image (H x W x 3 numpy array) the synthetic Modular frame of `seed` encodes losslessly
    (palette=1: the picture snapped to palette colours that encode_modular(..., palette=1) carries)."""
    import numpy as np
    lib = _lib()
    out = np.zeros((height, width, 3), np.uint8)
    if lib.jxs_modular_source_ex(width, height, seed, palette, out.ctypes.data) != 0:
        raise RuntimeError("synthetic source failed: " + lib.jxs_modular_last_error().decode())
    return out


def encode_modular(width, height, seed, rct=6, squeeze=0, tree_kind=1, source=None, palette=0) -> bytes:
    """One synthetic lossless Modular frame (8-bit RGB, group size 256). rct: 0 or 6 (YCoCg); squeeze: default
    Squeeze transform on/off; tree_kind: 0 single Gradient leaf, 1 property tree, 2 weighted-predictor tree,
    3 tree on properties of the previous channel (17, 19); palette: 1 = global palette transform over the colour
    channels (explicit entries + both implicit colour cubes, no delta entries; rct and squeeze must be 0).
    source: optional H x W x 3 uint8 array to encode instead of the procedural image."""
    lib = _lib()
    src = None
    if source is not None:
        import numpy as np
        source = np.ascontiguousarray(source, dtype=np.uint8)
        assert source.shape == (height, width, 3)
        src = source.ctypes.data
    cap = max(1 << 16, width * height * 4)
    buf = C.create_string_buffer(cap)
    n = lib.jxs_encode_modular_ex(width, height, seed, rct, squeeze, tree_kind, palette, src, buf, cap)
    if n < 0:
        raise RuntimeError("synthetic Modular encode failed: " + lib.jxs_modular_last_error().decode())
    if n > cap:
        buf = C.create_string_buffer(n)
        n = lib.jxs_encode_modular_ex(width, height, seed, rct, squeeze, tree_kind, palette, src, buf, n)
    return buf.raw[:n]


def _tree_words(tree):
    """A tree in BFS order: ("split", property, value) or ("leaf", predictor, offset, mul_log, mul_bits)."""
    words = [len(tree)]
    for n in tree:
        if n[0] == "split":
            words += [n[1] + 1, n[2], 0, 0, 0]
        else:
            words += [0, n[1], n[2], n[3], n[4]]
    return words


def _transform_words(transforms):
    words = [len(transforms)]
    for t in transforms:
        words.append(t["id"])
        if t["id"] == 0:
            words += [t["begin"], t["rct_type"]]
        elif t["id"] == 1:
            words += [t["begin"], t["num_c"], t["num_colors"], t["num_deltas"], t["predictor"]]
        else:
            words.append(len(t["squeezes"]))
            for sq in t["squeezes"]:
                words += [int(sq[0]), int(sq[1]), sq[2], sq[3]]
    return words


def encode_modular_tokens(spec) -> bytes:
    """One Modular frame written exactly as described; the writer predicts nothing and checks nothing (frames a decoder
    must refuse can be written). `spec` is a dict:
      width, height, group_shift (group size 128 << group_shift), grey, orientation (1..8), prefix (prefix codes
      instead of ANS), hybrid (split_exponent, msb, lsb) of every symbol cluster;
      tree: the global MA tree in BFS order, nodes ("split", property, value) / ("leaf", predictor, offset, mul_log,
      mul_bits); its leaf ids (BFS order) are the symbol contexts;
      sections: one per stream in TOC order without HfGlobal (global, then LF groups, then HF groups), each None (no
      bytes) or a dict with use_global_tree, wp (None: all_default, else the 11 fields p1c p2c p3ca..p3ce w0..w3),
      transforms (for the global section: the frame's global transforms) as dicts {"id": 0, "begin", "rct_type"},
      {"id": 1, "begin", "num_c", "num_colors", "num_deltas", "predictor"}, {"id": 2, "squeezes": [(horizontal,
      in_place, begin, num_c), ...]}, and tokens: None (the group header only) or a list of (context, u32 value);
      with tokens, "tree" is the local tree when use_global_tree is false."""
    words = [spec["width"], spec["height"], spec.get("group_shift", 1), int(spec.get("grey", 0)),
             spec.get("orientation", 1), int(spec.get("prefix", 0))] + list(spec.get("hybrid", (4, 2, 0)))
    words += _tree_words(spec["tree"])
    words.append(len(spec["sections"]))
    for s in spec["sections"]:
        if s is None:
            words.append(0)
            continue
        words.append(1 if s.get("tokens") is None else 2)
        words.append(int(s.get("use_global_tree", True)))
        wp = s.get("wp")
        words += [1] + [0] * 11 if wp is None else [0] + list(wp)
        words += _transform_words(s.get("transforms", []))
        if s.get("tokens") is not None:
            words += _tree_words(s.get("tree", []) if not s.get("use_global_tree", True) else [])
            toks = s["tokens"]
            words.append(len(toks))
            for c, v in toks:
                words += [c, v]
    lib = _lib()
    arr = (C.c_uint32 * len(words))(*[int(w) & 0xFFFFFFFF for w in words])
    cap = max(1 << 16, 8 * len(words))
    buf = C.create_string_buffer(cap)
    n = lib.jxs_encode_modular_tokens(arr, len(words), buf, cap)
    if n < 0:
        raise RuntimeError("token-level Modular encode failed: " + lib.jxs_modular_last_error().decode())
    if n > cap:
        buf = C.create_string_buffer(n)
        n = lib.jxs_encode_modular_tokens(arr, len(words), buf, n)
    return buf.raw[:n]
