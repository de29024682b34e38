"""Entropy-stage device time of one batch of many small frames: the shape where the lean entropy kernel has more frames
than resident CTAs, so that its schedule ends at one CTA per frame. Default: 800 synthetic frames of 768 x 768 (9 groups
each, 8 distinct ones repeated), device outputs. Prints one JSON line: the median entropy-stage time of the reruns, the
lean schedule of the first frame, the GPU and its power limit.

    python tools/entropy_schedule_times.py [--frames 800] [--size 768] [--reruns 7]

To compare two builds, run it from each tree in turn, alternating, in one session."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=800)
    ap.add_argument("--size", type=int, default=768)
    ap.add_argument("--reruns", type=int, default=7)
    args = ap.parse_args()
    import torch
    import jxl_rs_b200 as j
    import synth
    from jxl_rs_b200 import abi
    files = [synth.encode_synthetic(args.size, args.size, 500 + i, 0.5, 2, 1, 1) for i in range(8)]
    parsed = [j.ParsedFrame(f) for f in files]
    ctx = j.JxgContext(0)
    out = torch.empty((args.frames, args.size, args.size, 3), dtype=torch.uint8, device="cuda:0")
    b = j.Batch(ctx, args.frames)
    for i in range(args.frames):
        b.add(parsed[i % len(parsed)], out[i].data_ptr(), args.size * 3, abi.FORMAT_RGB_U8, True)
    b.set_profile(True)
    b.run()
    b.wait()
    times = []
    for _ in range(args.reruns):
        b.rerun_device()
        b.wait()
        times.append(b.stage_times()["entropy"])
    sched = b.entropy_schedule()["frames"][0] if hasattr(b, "entropy_schedule") else None
    stats = b.entropy_stats()
    b.close()
    ctx.close()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"tree": os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "frames": args.frames,
                      "size": args.size, "entropy_ms_median": round(statistics.median(times), 3),
                      "entropy_ms": [round(t, 3) for t in times], "lean_S": stats["lean_S"], "frame0": sched,
                      "gpu": gpu}))


if __name__ == "__main__":
    main()
