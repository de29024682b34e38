"""Device time of each transform-stage launch of one resident batch (bench workload: 3840x2160, profile 1, EPF 2), and
the varblocks of each transform class in the batch. Usage: python tools/transform_times.py [frames] [reruns]

Kernel times come from torch.profiler (CUDA activities) over `reruns` device reruns of the batch, one batch in flight;
the table is the mean per rerun. The classes are counted from each frame's transform map:
  reg8   types 0, 3, 12, 13      k_idct_small<0>, 8 lanes per varblock
  reg16  types 6, 7 (8 lanes), 4 (16 lanes)   k_idct_small<1>
  warp   other types up to 4x4 blocks         k_dequant_idct, one warp per varblock
  cta    larger than 4x4 blocks               k_dequant_idct, whole CTA per varblock"""
import ctypes as C
import os
import subprocess
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import bench
import jxl_rs_b200 as j
from jxl_rs_b200 import abi
from concurrent.futures import ThreadPoolExecutor

COV_X = [1, 1, 1, 1, 2, 4, 1, 2, 1, 4, 2, 4, 1, 1, 1, 1, 1, 1, 8, 4, 8, 16, 8, 16, 32, 16, 32]
COV_Y = [1, 1, 1, 1, 2, 4, 2, 1, 4, 1, 4, 2, 1, 1, 1, 1, 1, 1, 8, 8, 4, 16, 16, 8, 32, 32, 16]
KERNELS = ("k_block_plan", "k_idct_small<0>", "k_idct_small<1>", "k_dequant_idct")


def transform_class(t):
    if t in (0, 3, 12, 13):
        return "reg8"
    if t in (6, 7, 4):
        return "reg16"
    return "warp" if COV_X[t] <= 4 and COV_Y[t] <= 4 else "cta"


def class_counts(frame):
    d = frame.desc(abi.FORMAT_RGB_U8)[0]
    xb, yb = (frame.info.coded_width + 7) // 8, (frame.info.coded_height + 7) // 8
    tmap = np.ctypeslib.as_array(C.cast(d.transform_map, C.POINTER(C.c_uint8)), shape=(yb * xb,))
    hist = np.bincount(tmap[tmap >= 128] & 127, minlength=27)
    out = {"reg8": 0, "reg16": 0, "warp": 0, "cta": 0}
    for t, n in enumerate(hist):
        out[transform_class(t)] += int(n)
    return out


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    reruns = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    assert torch.cuda.is_available(), "transform_times.py needs a CUDA device"
    args = types.SimpleNamespace(frames=n, unique=0, width=3840, height=2160, distance=0.5, epf=2, profile=1)
    files = bench.make_frames(args, 0)
    with ThreadPoolExecutor(max_workers=16) as ex:
        frames = list(ex.map(j.ParsedFrame, files))
    counts = {"reg8": 0, "reg16": 0, "warp": 0, "cta": 0}
    for fr in frames:
        for k, v in class_counts(fr).items():
            counts[k] += v
    groups = sum(fr.info.num_groups for fr in frames)
    ctx = j.JxgContext(0)
    outs = [torch.empty((fr.height, fr.width, 3), dtype=torch.uint8, device="cuda:0") for fr in frames]
    b = j.Batch(ctx, n)
    for fr, o in zip(frames, outs):
        b.add(fr, o.data_ptr(), fr.width * 3, abi.FORMAT_RGB_U8, True)
    b.run()
    b.wait()
    b.rerun_device()  # warm
    b.wait()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reruns):
            b.rerun_device()
            b.wait()
    ms = {k: 0.0 for k in KERNELS}
    calls = {k: 0 for k in KERNELS}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                ms[k] += ev.self_device_time_total / 1000.0  # us -> ms
                calls[k] += ev.count
    b.close()
    ctx.close()
    print("card:", card())
    print(f"frames {n}, streams {groups}, reruns {reruns}")
    print("varblocks per batch:", counts)
    for k in KERNELS:
        print(f"  {k:18s} {ms[k] / reruns:8.3f} ms per batch  ({calls[k] // max(reruns, 1)} launches)")
    print(f"  transform stage    {sum(ms[k] for k in KERNELS[1:]) / reruns:8.3f} ms per batch (sum of the three launches)")


if __name__ == "__main__":
    main()
