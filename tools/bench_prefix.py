"""Prefix decode of VarDCT frames (jxg_parse_file_prefix + jxg_batch_add_parsed) on 64 synthetic 3840x2160 frames,
each cut at the end of HfGlobal (every group the LF image upsampled 8x), half way through the HF sections, and whole.

Reports, as one JSON line, per cut: the bytes of the files kept, and the device time of one batch of all frames
(RGB_U8, device outputs; median of CUDA events around `--reps` reruns after `--warmup`), also as a share of the
whole-file batch; with the card's name and power limit read in the same run.
--region: per cut, a centred 512x512 region and a centred 1920x1080 quarter of every frame
(jxg_batch_add_parsed_region) against the whole prefix decode at the same cut: device ms and H2D bytes per batch.
Usage: python tools/bench_prefix.py [--frames 64] [--reps 20] [--warmup 5] [--distance 0.5] [--region]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def batch_ms(ctx, frames, outs, reps, warmup, region=None, stats=None):
    """Median device ms of one batch of `frames` (each whole, or the region (x, y, w, h)); `stats` receives the
    batch's stats() of its first run."""
    import torch
    import jxl_rs_b200 as j
    b = j.Batch(ctx, len(frames))
    try:
        for fr, t in zip(frames, outs):
            b.add(fr, t.data_ptr(), (fr.width if region is None else region[2]) * 3, 0, True, region)
        b.run()
        b.wait()
        if stats is not None:
            stats.update(b.stats())
        st = torch.cuda.Stream()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for i in range(warmup + reps):
            with torch.cuda.stream(st):
                ev0.record(st)
                b.rerun_device(st.cuda_stream)
                ev1.record(st)
            ev1.synchronize()
            if i >= warmup:
                times.append(ev0.elapsed_time(ev1))
        b.wait()
    finally:
        b.close()
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--distance", type=float, default=0.5, help="synth.encode_synthetic distance (bench.py's 0.5)")
    ap.add_argument("--region", action="store_true", help="regions of each prefix against the whole prefix")
    a = ap.parse_args()
    import torch
    import jxl_rs_b200 as j
    import synth
    from tests import prefix_ref as pr
    synth.set_threads(os.cpu_count() or 1)
    files = [synth.encode_synthetic(3840, 2160, 1000 + i, a.distance) for i in range(a.frames)]
    starts = [pr.prefix_start(f) for f in files]
    cuts = {"hf_global_end": starts, "half_hf": [(s + len(f)) // 2 for s, f in zip(starts, files)],
            "whole": [len(f) for f in files]}
    res = {"frames": a.frames, "size": "3840x2160", "distance": a.distance, "card": card()}
    ctx = j.JxgContext(0)
    try:
        outs = [torch.empty((2160, 3840, 3), dtype=torch.uint8, device="cuda:0") for _ in files]
        if a.region:
            regions = {"whole": None, "512x512": (1664, 824, 512, 512), "1920x1080": (960, 540, 1920, 1080)}
            for name, cut in cuts.items():
                frames = [j.PrefixParsedFrame(f[:c]) for f, c in zip(files, cut)]
                res[name] = {}
                for rname, reg in regions.items():
                    st = {}
                    t = batch_ms(ctx, frames, outs, a.reps, a.warmup, reg, st)
                    res[name][rname] = {"device_ms_per_batch": t, "h2d_bytes_per_batch": st["h2d_bytes"]}
            print(json.dumps(res))
            return
        ms = {}
        for name, cut in cuts.items():
            frames = [j.PrefixParsedFrame(f[:c]) for f, c in zip(files, cut)]
            ms[name] = batch_ms(ctx, frames, outs, a.reps, a.warmup)
            res[name] = {"bytes": sum(cut), "share_of_bytes": sum(cut) / sum(len(f) for f in files),
                         "groups_without_pass": int(sum((fr.passes == 0).sum() for fr in frames)),
                         "device_ms_per_batch": ms[name]}
        ms["parse_file"] = batch_ms(ctx, [j.ParsedFrame(f) for f in files], outs, a.reps, a.warmup)
        res["whole_parse_file_device_ms"] = ms["parse_file"]
        for name in cuts:
            res[name]["vs_whole"] = ms[name] / ms["parse_file"]
    finally:
        ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
