"""Region decode against whole-frame decode on the bench workload (bench.make_frames: 64 x 3840x2160, EPF 2), four ways:
whole frames, one seeded random 224x224 crop per frame, one 1024x1024 crop per frame, and an 8 x 8 tiling of one
16384x16384 frame (EPF 3, bench.py --config 4's frame). Device-resident time per step (CUDA events around
rerun_device after warm-up, outputs in device memory), crops/s, output MP/s, entropy streams decoded and H2D bytes of
the upload; then an end-to-end run of the 224x224 crops through PipelinedDecoder (host parse of whole frames included).
One JSON line per run, each with the card's name and power limit read in the same process.

    python tools/bench_region.py [--steps 10] [--warmup 3] [--skip-16k]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": pl}


def device_step(ctx, items, steps, warmup):
    """items: (parsed frame, region or None). Device outputs; returns ms per rerun_device step and the batch counters."""
    import torch
    import jxl_rs_b200 as j
    from jxl_rs_b200 import abi
    b = j.Batch(ctx, len(items))
    bufs = []
    for pf, reg in items:
        w, h = (pf.width, pf.height) if reg is None else (reg[2], reg[3])
        t = torch.empty((h, w * 3), dtype=torch.uint8, device="cuda")
        bufs.append(t)
        b.add(pf, t.data_ptr(), w * 3, abi.FORMAT_RGB_U8, True, reg)
    b.run()
    b.wait()
    st = b.stats()
    es = b.entropy_stats()
    for _ in range(warmup):
        b.rerun_device()
    b.wait()
    # the events and the reruns on one stream of our own (stream handle 0 would select the context's stream)
    s = torch.cuda.Stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(s)
    for _ in range(steps):
        b.rerun_device(s.cuda_stream)
    e1.record(s)
    torch.cuda.synchronize()
    b.wait()
    b.close()
    ms = e0.elapsed_time(e1) / steps
    px = sum(t.numel() // 3 for t in bufs)
    return {"ms_per_step": round(ms, 3), "outputs_per_s": round(len(items) / ms * 1e3, 1), "output_mp_s": round(px / ms / 1e3, 1),
            "streams": es["lean"] + es["fast"] + es["slow"], "h2d_bytes": st["h2d_bytes"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-16k", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    import jxl_rs_b200 as j
    from jxl_rs_b200 import abi, decoder
    assert torch.cuda.is_available(), "bench_region measures on a CUDA device"
    info = card()
    wl = SimpleNamespace(frames=64, width=3840, height=2160, distance=0.5, epf=2, profile=1, unique=0, lf_tree=0)
    files = bench.make_frames(wl, 0)
    pfs = [j.ParsedFrame(f) for f in files]
    rng = np.random.default_rng(7)

    def crops(size):
        return [(int(rng.integers(0, 3840 - size + 1)), int(rng.integers(0, 2160 - size + 1)), size, size) for _ in pfs]

    ctx = j.JxgContext(0)
    runs = [("full", [(pf, None) for pf in pfs]), ("crop224", list(zip(pfs, crops(224)))),
            ("crop1024", list(zip(pfs, crops(1024))))]
    for name, items in runs:
        r = device_step(ctx, items, args.steps, args.warmup)
        print(json.dumps({"run": name, "workload": "64 x 3840x2160 EPF 2", **r, **info}), flush=True)
    # end to end: host parse of whole frames + region decode, through the serving entry point
    c224 = crops(224)
    outs = [torch.empty((224, 224 * 3), dtype=torch.uint8).pin_memory() for _ in files]
    dec = decoder.PipelinedDecoder(0, depth=3)
    try:
        dec.decode(files, [(o.data_ptr(), 224 * 3) for o in outs], abi.FORMAT_RGB_U8, regions=c224)  # warm-up
        t0 = time.perf_counter()
        for _ in range(args.steps):
            dec.submit(files, [(o.data_ptr(), 224 * 3) for o in outs], abi.FORMAT_RGB_U8, regions=c224)
        dec.drain()
        dt = (time.perf_counter() - t0) / args.steps
    finally:
        dec.close()
    print(json.dumps({"run": "crop224_pipelined", "workload": "64 x 3840x2160 EPF 2, host parse included",
                      "ms_per_step": round(dt * 1e3, 2), "outputs_per_s": round(len(files) / dt, 1),
                      "host_cores": decoder.effective_cpus(), **info}), flush=True)
    del pfs
    if not args.skip_16k:
        wl16 = SimpleNamespace(frames=1, width=16384, height=16384, distance=0.5, epf=3, profile=1, unique=0, lf_tree=0)
        big = j.ParsedFrame(bench.make_frames(wl16, 0)[0], decoder.effective_cpus())
        tiles = [(x * 2048, y * 2048, 2048, 2048) for y in range(8) for x in range(8)]
        for name, items in (("16k_full", [(big, None)]), ("16k_tiles8x8", [(big, t) for t in tiles])):
            r = device_step(ctx, items, args.steps, args.warmup)
            print(json.dumps({"run": name, "workload": "1 x 16384x16384 EPF 3", **r, **info}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
