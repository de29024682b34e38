"""Entropy-stage device time (block plan + entropy kernel) of the batches that do not take the lean kernel, which bench.py
does not run: prefix-coded frames (k_entropy_fast), LZ77 frames and multi-pass frames (k_entropy). Each batch's route is
asserted through Batch.entropy_stats(). Usage: python tools/entropy_times.py [reruns]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import statistics
import torch
import jxl_rs_b200 as j
import synth
from jxl_rs_b200 import abi
from concurrent.futures import ThreadPoolExecutor
from tests import test_vardct_ref as T
reruns = int(sys.argv[1]) if len(sys.argv) > 1 else 10


def encode(n, entropy):
    with ThreadPoolExecutor(max_workers=16) as ex:
        return list(ex.map(lambda i: synth.encode_synthetic(1920, 1080, 100 + i, 0.5, 2, 1, 1, entropy=entropy), range(n)))


BATCHES = [
    ("prefix 64x1920x1080", "fast", lambda: encode(64, 1)),
    ("lz77 64x1920x1080", "slow", lambda: encode(32, 2) + encode(32, 3)),
    ("passes2 256x320x288", "slow", lambda: [T.model("passes2_wrap")[1]] * 256),
]

ctx = j.JxgContext(0)
for name, route, make in BATCHES:
    with ThreadPoolExecutor(max_workers=16) as ex:
        frames = list(ex.map(j.ParsedFrame, make()))
    outs = [torch.empty((fr.height, fr.width, 3), dtype=torch.uint8, device="cuda:0") for fr in frames]
    b = j.Batch(ctx, len(frames))
    for fr, o in zip(frames, outs):
        b.add(fr, o.data_ptr(), fr.width * 3, abi.FORMAT_RGB_U8, True)
    b.set_profile(True)
    b.run(); b.wait()
    st = b.entropy_stats()
    assert st[route] > 0 and st[route] == st["lean"] + st["fast"] + st["slow"], (name, st)
    ms = []
    for _ in range(reruns):
        b.rerun_device(); b.wait()
        ms.append(b.stage_times()["entropy"])
    b.close()
    print(f"{name}: {route} streams {st[route]}, entropy ms min {min(ms):.3f} median {statistics.median(ms):.3f}", flush=True)
ctx.close()
