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
                                                 C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
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
        _LIB.jxs_encode_modular_lz77.restype = C.c_int64
        _LIB.jxs_encode_modular_lz77.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32,
                                                 C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t]
        _LIB.jxs_modular_lz77_census.argtypes = [C.c_void_p]
        _LIB.jxs_modular_lz77_census.restype = None
        _LIB.jxs_encode_vardct_tokens.restype = C.c_int64
        _LIB.jxs_encode_vardct_tokens.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    return _LIB


def encode_synthetic(width, height, seed, distance=1.0, epf_iters=2, gab=1, profile=1, lf_tree=0, entropy=0, orientation=1,
                     colour=0, dequant=None, x_qm_scale=3, b_qm_scale=2, header=None, lf_extra_precision=0,
                     skip_lf_smoothing=False, lf_entropy=0) -> bytes:
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
    quantised with the tables the decoder computes from what is written.
    header: None (default fields) or a dict of fields written as given, every float a 16-bit f16 pattern (see
    _header_words); the writer checks nothing, so frames the decoder must refuse can be written. The source picture
    is converted with the opsin matrix and biases written, and quantised with the colour correlation (factor, bases,
    LF factors, tile maps clamped to i8) the decoder derives, so the round trip holds as for default headers; a
    non-finite f16 falls back to the default value there (the decoder refuses such a frame). Gaborish and EPF are not
    inverted by the writer, as with the default weights.
    lf_extra_precision: 0..3, written in every LF group with the quantised LF samples unchanged (the decoded LF image is
    scaled by 2^-lf_extra_precision, a valid frame of a different picture). skip_lf_smoothing: sets the frame flag that
    turns the adaptive LF smoothing off. lf_entropy: code of the LF image's pixel symbols, as `entropy` (0 ANS, 1 prefix
    codes, 2 / 3 the same with LZ77 copies at plain distances)."""
    profile = ((profile & 0xff) | ((lf_tree & 1) << 8) | ((entropy & 3) << 9) | (((orientation - 1) & 7) << 12)
               | ((colour & 15) << 16) | ((lf_extra_precision & 3) << 20) | ((1 if skip_lf_smoothing else 0) << 22)
               | ((lf_entropy & 3) << 23))
    lib = _lib()
    words = _dequant_words(dequant)
    arr = (C.c_uint32 * max(1, len(words)))(*[w & 0xFFFFFFFF for w in words])
    hwords = _header_words(header)
    harr = (C.c_uint32 * max(1, len(hwords)))(*[int(w) & 0xFFFFFFFF for w in hwords])

    def run(buf, cap):
        if not words and not hwords and (x_qm_scale, b_qm_scale) == (3, 2):
            return lib.jxs_encode_synthetic(width, height, seed, distance, epf_iters, gab, profile, buf, cap)
        return lib.jxs_encode_synthetic_ex(width, height, seed, distance, epf_iters, gab, profile, x_qm_scale, b_qm_scale,
                                           arr, len(words), harr, len(hwords), buf, cap)
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


def _header_words(header):
    """The flat u32 array of jxs_encode_synthetic_ex's header. Keys of `header`, each optional (absent: not custom):
      gab: the six Gaborish weights x w1, x w2, y w1, y w2, b w1, b w2 (written when gab = 1);
      sharp: the 8 entries of epf_sharp_lut; weight: epf_channel_scale X, Y, B and the two zeroflush values (parsed
      and ignored); sigma: epf_quant_mul, epf_pass0_sigma_scale, epf_pass2_sigma_scale, epf_border_sad_mul (the EPF
      groups are written when epf_iters > 0);
      color: {"factor": (selector 0..3, bits: 84 / 256 / bits + 2 (8 bits) / bits + 258 (16 bits)), "base_x",
      "base_b", "ytox_lf", "ytob_lf" (integers -128..127)};
      opsin: {"matrix": 9, "biases": 3, "quant_biases": 4};
      cfl: (ytox, ytob), each one integer per 64x64 tile in raster order, any i32 (the decoder clamps to i8)."""
    if not header:
        return []
    words = []
    for key, n in (("gab", 6), ("sharp", 8), ("weight", 5), ("sigma", 4)):
        v = header.get(key)
        assert v is None or len(v) == n, key
        words += [0] * (n + 1) if v is None else [1] + [int(x) & 0xFFFF for x in v]
    cc = header.get("color")
    if cc is None:
        words += [0, 0, 0, 0, 0, 128, 128]
    else:
        sel, bits = cc.get("factor", (0, 0))
        words += [1, sel, bits, cc.get("base_x", 0), cc.get("base_b", 0x3C00), cc.get("ytox_lf", 0) + 128,
                  cc.get("ytob_lf", 0) + 128]
    op = header.get("opsin")
    if op is None:
        words += [0] * 17
    else:
        assert len(op["matrix"]) == 9 and len(op["biases"]) == 3 and len(op["quant_biases"]) == 4
        words += [1] + [int(x) & 0xFFFF for x in list(op["matrix"]) + list(op["biases"]) + list(op["quant_biases"])]
    cfl = header.get("cfl")
    if cfl is None:
        words.append(0)
    else:
        ytox, ytob = (list(_flat(m)) for m in cfl)
        assert len(ytox) == len(ytob)
        words += [len(ytox)] + [int(v) for v in ytox] + [int(v) for v in ytob]
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


def encode_modular(width, height, seed, rct=6, squeeze=0, tree_kind=1, source=None, palette=0, lz77=0) -> bytes:
    """One synthetic lossless Modular frame (8-bit RGB, group size 256). rct: 0 or 6 (YCoCg); squeeze: default
    Squeeze transform on/off; tree_kind: 0 single Gradient leaf, 1 property tree, 2 weighted-predictor tree,
    3 tree on properties of the previous channel (17, 19); palette: 1 = global palette transform over the colour
    channels (explicit entries + both implicit colour cubes, no delta entries; rct and squeeze must be 0).
    source: optional H x W x 3 uint8 array to encode instead of the procedural image.
    lz77: 0 no LZ77; 1 run-length copies in the group streams (every copy at distance 1, the shape libjxl's fastest
    lossless mode writes); 2 general copies (special distances relative to the stream's widest channel, plain
    distances, copies across row ends and channels, copies the decoder clamps). lz77_census() describes the copies."""
    lib = _lib()
    src = None
    if source is not None:
        import numpy as np
        source = np.ascontiguousarray(source, dtype=np.uint8)
        assert source.shape == (height, width, 3)
        src = source.ctypes.data
    cap = max(1 << 16, width * height * 4)
    buf = C.create_string_buffer(cap)

    def run(buf, cap):
        if lz77:
            return lib.jxs_encode_modular_lz77(width, height, seed, rct, squeeze, tree_kind, palette, lz77, src, buf, cap)
        return lib.jxs_encode_modular_ex(width, height, seed, rct, squeeze, tree_kind, palette, src, buf, cap)
    n = run(buf, cap)
    if n < 0:
        raise RuntimeError("synthetic Modular encode failed: " + lib.jxs_modular_last_error().decode())
    if n > cap:
        buf = C.create_string_buffer(n)
        n = run(buf, n)
    return buf.raw[:n]


LZ77_CENSUS_KEYS = ("copies", "special", "plain", "cross_channel", "clamped", "max_distance", "max_stream")


def lz77_census():
    """What the last LZ77 encode of this thread wrote (encode_modular with lz77 > 0, encode_modular_tokens with
    spec["lz77"]): copies, copies with special / plain distances, copies crossing a channel boundary, copies whose
    distance the decoder clamps to the symbols decoded so far, the longest distance copied from, the longest stream."""
    out = (C.c_uint64 * 7)()
    _lib().jxs_modular_lz77_census(out)
    return dict(zip(LZ77_CENSUS_KEYS, list(out)))


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
      with tokens, "tree" is the local tree when use_global_tree is false.
    lz77 (optional): a dict with min_symbol (default 224), min_length (3), length (hybrid config of the copy lengths,
    (0, 0, 0)), mode (1 run-length, 2 general: see encode_modular), multipliers (per section, the widest channel of its
    stream: the unit of the special distances) and fault (None, or (1, section): that stream starts with a copy,
    (2, section): its first copy has a length that overflows). The decoded values are those of the token lists."""
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
    lz = spec.get("lz77")
    if lz:
        fault = lz.get("fault") or (0, 0)
        mult = list(lz["multipliers"])
        assert len(mult) == len(spec["sections"])
        words += [lz.get("min_symbol", 224), lz.get("min_length", 3)] + list(lz.get("length", (0, 0, 0)))
        words += [lz["mode"], fault[0], fault[1]] + mult
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


def encode_vardct_tokens(spec) -> bytes:
    """One VarDCT frame whose AC coefficient streams hold exactly the given tokens; the writer predicts nothing and checks
    nothing (frames a decoder must refuse can be written). The image metadata, the LF quantisation and the
    dequantisation matrices are the defaults; so are the colour correlation, the opsin fields, the filter weights and
    the CfL maps unless `header` / `cfl` give them. `spec` is a dict:
      width, height; shifts: one per pass (1..11 passes), the last one 0;
      bcm: None (the default BlockContextMap) or {"lf": [X, Y, B threshold lists], "qf": [thresholds as decoded, >= 1],
      "map": block context per (channel, order, qf bucket, LF bucket)};
      lf: (3, yb, xb) quantised LF integers of the channels X, Y, B; varblocks: (bx, by, transform, raw_quant) tiling
      the frame; num_histograms;
      passes: per pass {"selector": 0..3, "used_orders": the 13 bits of selector 3, "perms": {(order, channel):
      permutation of 64 * num_blocks entries, the first num_blocks fixed}, "cmap": context -> cluster, "cfgs": hybrid
      (split_exponent, msb, lsb) per cluster, "log_alpha": the smallest ANS alphabet (log2), "prefix": prefix codes,
      "lz77": None or (min_symbol, min_length)};
      sections: per pass, per group: (histogram index, [(context, u32 value), ...]);
      header (optional): the header fields of encode_synthetic's `header` dict (_header_words), written as given; its
      restoration filter groups apply to the frame's Gaborish + EPF 2 header;
      cfl (optional): (ytox, ytob) CfL tile maps, one i32 per 64x64 tile in raster order (default: zeros)."""
    import numpy as np
    header = dict(spec.get("header") or {})
    if spec.get("cfl") is not None:
        header["cfl"] = spec["cfl"]
    hwords = _header_words(header)
    words = [len(hwords)] + hwords + [spec["width"], spec["height"], len(spec["shifts"])] + list(spec["shifts"][:-1])
    bcm = spec.get("bcm")
    if bcm is None:
        words.append(0)
    else:
        words.append(1)
        for thr in bcm["lf"]:
            words += [len(thr)] + list(thr)
        words += [len(bcm["qf"])] + list(bcm["qf"])
        words += [len(bcm["map"])] + list(bcm["map"])
    lf = np.asarray(spec["lf"], np.int64)
    words += lf.transpose(1, 2, 0).reshape(-1).tolist()
    words.append(len(spec["varblocks"]))
    for vb in spec["varblocks"]:
        words += list(vb)
    words.append(spec["num_histograms"])
    for p in spec["passes"]:
        words += [p.get("selector", 2), p.get("used_orders", 0), len(p.get("perms", {}))]
        for (o, c), perm in p.get("perms", {}).items():
            words += [o, c, len(perm)] + list(perm)
        words += [len(p["cmap"])] + list(p["cmap"]) + [len(p["cfgs"])]
        for cfg in p["cfgs"]:
            words += list(cfg)
        lz = p.get("lz77")
        words += [p.get("log_alpha", 5), int(p.get("prefix", 0)), int(lz is not None)] + list(lz or (224, 3))
    for hist, toks in spec["sections"]:
        words += [hist, len(toks)]
        for c, v in toks:
            words += [c, v]
    lib = _lib()
    arr = np.asarray([int(w) & 0xFFFFFFFF for w in words], np.uint32)
    cap = max(1 << 16, 8 * len(words))
    buf = C.create_string_buffer(cap)
    n = lib.jxs_encode_vardct_tokens(arr.ctypes.data, len(words), buf, cap)
    if n < 0:
        raise RuntimeError("token-level VarDCT encode failed: " + lib.jxs_last_error().decode())
    if n > cap:
        buf = C.create_string_buffer(n)
        n = lib.jxs_encode_vardct_tokens(arr.ctypes.data, len(words), buf, n)
    return buf.raw[:n]
