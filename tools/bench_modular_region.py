"""Device time of Modular region decode against the whole frame (jxg_modular_batch_add_region).

Per workload: one batch is built and run once, then rerun on the device (inputs resident); the time is the median over
the reruns of CUDA events around one rerun, after warm-up reruns. Prints one JSON line per workload, with the card's
name and power limit read in the same run.
  config5      8 x 4096^2 synth.encode_modular(4096, 4096, seed, 6, 0, 1): whole frames, one random 224^2 crop per
               frame, one random 1024^2 crop per frame
  issue865     issue865_large_toc.jxl (5249 x 5377, 1806 groups): whole frame, one 256^2 tile
  squeeze      grayscale_public_university.jxl: a 256^2 crop at the top left, one at the bottom right (the cone of a
               Squeeze frame reaches the top-left corner of every level)
Usage: python tools/bench_modular_region.py [--reps 30] [--warmup 5]"""
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


def time_batch(ctx, items, reps, warmup):
    """items: [(ModularParsedFrame, region or None)]. Median device ms of one rerun, and the streams decoded."""
    import numpy as np
    import torch
    import jxl_rs_b200 as j
    b = j.ModularBatch(ctx)
    outs = []
    try:
        for fr, reg in items:
            w, h = (fr.width, fr.height) if reg is None else (reg[2], reg[3])
            t = torch.empty((h, w, 3), dtype=torch.uint8, device="cuda:0")
            outs.append(t)
            b.add(fr, t.data_ptr(), w * 3, True, region=reg)
        walks = b.walk_stats()
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
        b.wait()
    finally:
        b.close()
    rects = walks["generic"] + walks["single_leaf"] + sum(walks["by_property"].values())
    return float(np.median(ms)), rects


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch
    import jxl_rs_b200 as j
    import synth
    assert torch.cuda.is_available(), "this benchmark measures the GPU; there is no CPU fallback"
    gpu = card()
    ctx = j.JxgContext(0)
    rng = np.random.default_rng(5)

    def crop(fr, n):
        return (int(rng.integers(0, fr.width - n + 1)), int(rng.integers(0, fr.height - n + 1)), n, n)

    def report(workload, items):
        ms, rects = time_batch(ctx, items, a.reps, a.warmup)
        print(json.dumps({"workload": workload, "device_ms": round(ms, 4), "frames": len(items),
                          "stream_rects_decoded": rects, "gpu": gpu}), flush=True)

    frames = [j.ModularParsedFrame(synth.encode_modular(4096, 4096, 100 + i, 6, 0, 1)) for i in range(8)]
    report("config5_whole", [(f, None) for f in frames])
    report("config5_crop224", [(f, crop(f, 224)) for f in frames])
    report("config5_crop1024", [(f, crop(f, 1024)) for f in frames])
    gold = os.path.join(ROOT, "tests", "golden", "jxl")
    big = j.ModularParsedFrame(open(os.path.join(gold, "issue865_large_toc.jxl"), "rb").read())
    report("issue865_whole", [(big, None)])
    report("issue865_tile256", [(big, crop(big, 256))])
    sq = j.ModularParsedFrame(open(os.path.join(gold, "grayscale_public_university.jxl"), "rb").read())
    report("squeeze_whole", [(sq, None)])
    report("squeeze_top_left256", [(sq, (0, 0, 256, 256))])
    report("squeeze_bottom_right256", [(sq, (sq.width - 256, sq.height - 256, 256, 256))])
    ctx.close()


if __name__ == "__main__":
    main()
