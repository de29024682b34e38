"""Device time of XYB (lossy) Modular frames: 8 synthetic 4096 x 4096 XYB frames with the default Squeeze, decoded into
RGB u8 (and RGB f16) on the device (jxg_modular_batch_add_output).

One batch is built and run once, then rerun on the device (inputs resident); the time is the median over the reruns
of CUDA events around one rerun, after warm-up reruns. The share of the XYB store (k_xyb_store<true>: conversion,
output stage and store) is its kernel time over all kernel time of one profiled rerun, taken in a separate pass with
torch.profiler. Prints one JSON line per workload, with the card's name and power limit read in the same run.
Usage: python tools/bench_modular_xyb.py [--reps 20] [--warmup 3] [--frames 8] [--size 4096]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run(ctx, frames, fmt, reps, warmup):
    """Median device ms of one rerun, and the XYB store's share of the kernel time of one profiled rerun."""
    import numpy as np
    import torch
    import jxl_rs_b200 as j
    from jxl_rs_b200 import abi
    b = j.ModularBatch(ctx)
    outs = []
    try:
        for fr in frames:
            t = torch.empty((fr.height, fr.width * abi.BYTES_PER_PIXEL[fmt]), dtype=torch.uint8, device="cuda:0")
            outs.append(t)
            b.add(fr, t.data_ptr(), t.shape[1], True, fmt=fmt)
        b.run()
        b.wait()
        st = torch.cuda.Stream()  # a stream of its own: rerun_device(0) would run on the context's stream
        ms = []
        with torch.cuda.stream(st):
            for _ in range(warmup):
                b.rerun_device(st.cuda_stream)
            for _ in range(reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                b.rerun_device(st.cuda_stream)
                e1.record(st)
                e1.synchronize()
                ms.append(e0.elapsed_time(e1))
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                b.rerun_device(st.cuda_stream)
                st.synchronize()
        b.wait()
    finally:
        b.close()
    total = store = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if not e.key.startswith(("Memcpy", "Memset")):
            total += t
            if "k_xyb_store<true>" in e.key:
                store += t
    return float(np.median(ms)), (store / total if total else float("nan"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--size", type=int, default=4096)
    a = ap.parse_args()
    import torch
    import jxl_rs_b200 as j
    import synth
    from jxl_rs_b200 import abi
    assert torch.cuda.is_available(), "this benchmark measures the GPU; there is no CPU fallback"
    gpu = card()
    ctx = j.JxgContext(0)
    n = a.size
    frames = [j.ModularParsedFrame(synth.encode_modular(n, n, 200 + i, rct=0, squeeze=1, xyb={}))
              for i in range(a.frames)]
    mpix = a.frames * n * n / 1e6
    for name, fmt in (("rgb_u8", abi.FORMAT_RGB_U8), ("rgb_f16", abi.FORMAT_RGB_F16)):
        ms, share = run(ctx, frames, fmt, a.reps, a.warmup)
        print(json.dumps({"workload": f"xyb_squeeze_{n}_{name}", "frames": a.frames, "device_ms": round(ms, 3),
                          "mp_per_s": round(mpix / (ms / 1e3), 1), "xyb_store_share": round(share, 4), "gpu": gpu}),
              flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
