"""LZ77 group streams on the Modular device path: 8 x 4096x4096 frames of one flat-region picture (rectangles, a
gradient band, text-like strokes) written without copies (lz77=0), with run-length copies (1, libjxl's fastest lossless
mode) and with general copies (2), decoded at 1, 2 and 4 lanes per warp. Prints one JSON line per (lz77, lanes):
device-resident MP/s, decode-kernel ms, LZ77 window bytes, bytes per frame; the card and its power limit first.
With --parent DIR it then runs `bench.py --config 5` (no LZ77) from DIR and from this tree, alternated, so that the
copy-free path can be compared against the parent commit within one run.
Usage: python tools/bench_modular_lz77.py [--frames 8] [--reps 5] [--parent DIR] [--config5-rounds 3]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def flat_picture(w, h, seed=0):
    import numpy as np
    rng = np.random.default_rng(seed)
    img = np.full((h, w, 3), 236, np.uint8)
    for _ in range(max(4, (w * h) >> 14)):
        x0, y0 = int(rng.integers(0, w)), int(rng.integers(0, h))
        x1, y1 = min(w, x0 + int(rng.integers(8, max(9, w // 3)))), min(h, y0 + int(rng.integers(8, max(9, h // 3))))
        img[y0:y1, x0:x1] = rng.integers(0, 256, 3)
    band = slice(h // 3, h // 3 + max(1, h // 10))
    img[band, :, 0] = (np.arange(w) * 255 // max(1, w - 1)).astype(np.uint8)[None, :]
    for y in range(5, h, 23):
        img[y, (np.arange(w) % 7) < 4] = 20
    return img


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def lz77_rows(args):
    import numpy as np
    import torch
    import jxl_rs_b200 as j
    import synth
    W = H = 4096
    src = flat_picture(W, H)
    ctx = j.JxgContext(0)
    outs = [torch.empty((H, W, 3), dtype=torch.uint8, device="cuda:0") for _ in range(args.frames)]
    for lz in (0, 1, 2):
        data = synth.encode_modular(W, H, 1, source=src, lz77=lz)
        frames = [j.ModularParsedFrame(data) for _ in range(args.frames)]
        for lanes in (1, 2, 4):
            b = j.ModularBatch(ctx, lanes)
            for fr, o in zip(frames, outs):
                b.add(fr, o.data_ptr(), W * 3, True)
            lzst = b.lz77_stats()
            b.run()
            b.wait()
            ok = all(np.array_equal(o.cpu().numpy(), src) for o in outs[:2])
            dev, dec = [], []
            for _ in range(args.reps):
                b.rerun_device()
                b.wait()
                st = b.stats()
                dev.append(st["device_ms"])
                dec.append(st["decode_ms"])
            b.close()
            dev.sort()
            dec.sort()
            print(json.dumps({"lz77": lz, "lanes_per_warp": lanes, "frames": args.frames,
                              "mp_per_s_device": round(args.frames * W * H / dev[len(dev) // 2] / 1e3, 1),
                              "device_ms_median": round(dev[len(dev) // 2], 2), "device_ms_min": round(dev[0], 2),
                              "device_ms_max": round(dev[-1], 2), "decode_kernel_ms_median": round(dec[len(dec) // 2], 2),
                              "window_bytes": lzst["window_bytes"], "lz77_streams": lzst["lz77_streams"],
                              "rle_streams": lzst["rle_streams"], "bytes_per_frame": len(data), "bit_exact": ok}),
                  flush=True)
    ctx.close()


def config5(args):
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--config", "5", "--steps", str(args.steps), "--warmup", str(args.warmup)]
    for r in range(args.config5_rounds):
        for name, d in (("parent", args.parent), ("branch", ROOT)):
            p = subprocess.run(cmd, cwd=d, capture_output=True, text=True)
            line = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
            res = json.loads(line[-1]) if line else {"error": p.stderr[-400:]}
            print(json.dumps({"config5": name, "round": r, "value": res.get("value"), "unit": res.get("unit"),
                              "device_resident": res.get("device_resident", res.get("detail"))}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parent", default=None, help="a built tree of the parent commit, for the bench.py --config 5 A/B")
    ap.add_argument("--config5-rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    lz77_rows(args)
    if args.parent:
        config5(args)


if __name__ == "__main__":
    main()
