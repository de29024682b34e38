"""Restatements behind the prefix-decode tests (tests/test_prefix.py, tests/test_gpu_prefix.py): which passes each HF
group of a cut file decodes (frame_info.rs:302-328, 548-565), and the float64 Upsample8x that fills the groups with none
(frame/decode.rs:51-150 upsample_lf_group, render/stages/upsample.rs)."""
import ctypes as C
import json
import os
import struct

import numpy as np

import jxl_rs_b200 as j
from jxl_rs_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = os.path.join(HERE, "golden", "jxl")


def bare_codestream(data: bytes) -> bytes:
    """The codestream of a .jxl file: the file itself, or the jxlc / jxlp payloads of a container in order."""
    if data[:2] == b"\xff\x0a":
        return data
    out, pos = b"", 0
    while pos + 8 <= len(data):
        size, kind = struct.unpack(">I4s", data[pos:pos + 8])
        head = 8
        if size == 1:
            size, head = struct.unpack(">Q", data[pos + 8:pos + 16])[0], 16
        end = len(data) if size == 0 else pos + size
        if kind == b"jxlc":
            out += data[pos + head:end]
        elif kind == b"jxlp":
            out += data[pos + head + 4:end]
        pos = end
    return out


def fixture(name):
    return bare_codestream(open(os.path.join(FIXTURES, name), "rb").read())


def hf_sections(data):
    """(offsets, lengths) of the HF sections of a whole bare codestream, [passes][groups], from the full parse."""
    fr = j.ParsedFrame(data)
    d, _, off, ln, n = fr.desc(abi.FORMAT_RGB_U8)
    off = np.ctypeslib.as_array(C.cast(off, C.POINTER(C.c_uint64)), shape=(n,)).astype(np.int64)
    ln = np.ctypeslib.as_array(C.cast(ln, C.POINTER(C.c_uint32)), shape=(n,)).astype(np.int64)
    p, g = fr.info.num_passes, fr.info.num_groups
    return off.reshape(p, g), ln.reshape(p, g)


def group_passes(off, ln, cut):
    """Rule of check_group: the longest run of passes from pass 0 whose sections lie wholly inside the first `cut` bytes."""
    inside = off + ln <= cut
    k = np.zeros(off.shape[1], np.uint8)
    for g in range(off.shape[1]):
        while k[g] < off.shape[0] and inside[k[g], g]:
            k[g] += 1
    return k


def prefix_code(data):
    try:
        j.PrefixParsedFrame(data)
        return 0
    except abi.JxgError as e:
        return e.code


def prefix_start(data):
    """The shortest prefix the prefix parse accepts (binary search; accepted prefixes are upward closed, checked by the
    callers)."""
    lo, hi = 1, len(data)
    while lo < hi:
        mid = (lo + hi) // 2
        if prefix_code(data[:mid]) == 0:
            hi = mid
        else:
            lo = mid + 1
    return lo


def default_weights8():
    return np.array(json.load(open(os.path.join(HERE, "golden", "upsample8_weights.json")))["weights8"], np.float64)


def f16_bits_to_float(bits):
    return np.array(bits, np.uint16).view(np.float16).astype(np.float64)


def upsample8_kernel(weights):
    """Upsample8x::new (upsample.rs:21-69): k[oy, ox, ky, kx]."""
    k = np.zeros((8, 8, 5, 5))
    for i in range(20):
        for jj in range(20):
            y, x = min(i, jj), max(i, jj)
            w = weights[20 * y - y * (y - 1) // 2 + x - y]
            k[jj // 5, i // 5, jj % 5, i % 5] = w
            k[7 - jj // 5, i // 5, 4 - jj % 5, i % 5] = w
            k[jj // 5, 7 - i // 5, jj % 5, 4 - i % 5] = w
            k[7 - jj // 5, 7 - i // 5, 4 - jj % 5, 4 - i % 5] = w
    return k


def mirror(v, s):
    while v < 0 or v >= s:
        v = -v - 1 if v < 0 else 2 * s - v - 1
    return v


def upsample_lf_group(lf, gx, gy, kernel):
    """upsample_lf_group for one channel of one 256x256 group, in float64: the LF plane lf (yb, xb) -> the group's
    (8 * rows, 8 * cols) pixels. The row buffer is restated literally, its zero-initialised slots included."""
    lh, lw = lf.shape
    lx0, ly0 = gx * 32, gy * 32
    lx1 = min(lx0 + 32, lw)
    start_x, end_x = max(lx0 - 2, 0), min(lx1 + 2, lw)
    cw = end_x - start_x
    save_start = 2 if start_x == lx0 else 0
    save_end = save_start + cw
    xs, ys = lx1 - lx0, min(32, lh - ly0)
    out = np.zeros((ys * 8, xs * 8))
    storage = [np.zeros(lw + 40) for _ in range(5)]  # reused across rows, as the reference's buffers are
    for y in range(ys):
        for dy in range(-2, 3):
            st = storage[dy + 2]
            st[save_start:save_end] = lf[mirror(ly0 + y + dy, lh), start_x:end_x]
            if start_x == lx0:
                st[0] = st[2 + mirror(-2, cw)]
                st[1] = st[2 + mirror(-1, cw)]
            if end_x == lx1:
                st[save_end] = st[save_start + mirror(save_end, save_end)]
                st[save_end + 1] = st[save_start + mirror(save_end + 1, save_end)]
        win = np.stack(storage)  # 5 x buffer
        for x in range(xs):
            w = win[:, x:x + 5]
            mn, mx = w.min(), w.max()
            v = np.einsum("abkl,kl->ab", kernel, w)
            out[y * 8:(y + 1) * 8, x * 8:(x + 1) * 8] = np.clip(v, mn, mx)
    return out
