"""1:8 thumbnails of VarDCT frames (jxg_lf_parse_file + jxg_modular_batch_add_lf) on 64 synthetic 3840x2160 frames.

Reports, as one JSON line:
  - bytes: the prefix of each file the thumbnail parse needs (the shortest prefix it accepts, by binary search) as a share
    of the file size; computed without a device;
  - host parse time per frame on one core (median over the frames, each parsed `--reps` times): jxg_lf_parse_file
    against jxg_parse_file;
  - device time of one thumbnail batch of all frames (RGB_U8, device outputs; median of CUDA events around
    `--reps` reruns after `--warmup`) and thumbnails per second, with the card's name and power limit read in the same
    run.
--cpu-only stops after the byte counts and the host parse times and needs no device.
Usage: python tools/bench_lf_thumbnail.py [--frames 64] [--reps 20] [--warmup 5] [--cpu-only] [--distance 1.0]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def lf_prefix(data):
    """Length of the shortest prefix of a bare codestream that jxg_lf_parse_file accepts."""
    import jxl_rs_b200 as j
    from jxl_rs_b200 import abi

    def ok(n):
        try:
            j.LfParsedFrame(data[:n])
            return True
        except abi.JxgError:
            return False
    lo, hi = 1, len(data)
    while lo < hi:
        mid = (lo + hi) // 2
        if ok(mid):
            hi = mid
        else:
            lo = mid + 1
    return lo


def parse_ms(cls, data, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        cls(data)
        t.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cpu-only", action="store_true")
    ap.add_argument("--distance", type=float, default=1.0, help="synth.encode_synthetic distance (bench.py uses 0.5)")
    a = ap.parse_args()
    import jxl_rs_b200 as j
    import synth
    synth.set_threads(os.cpu_count() or 1)
    files = [synth.encode_synthetic(3840, 2160, 1000 + i, a.distance) for i in range(a.frames)]
    res = {"frames": a.frames, "size": "3840x2160", "distance": a.distance}
    read = sum(lf_prefix(f) for f in files)
    total = sum(len(f) for f in files)
    res["bytes_read"], res["bytes_total"], res["read_share"] = read, total, read / total
    os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})  # one core
    res["host_parse_ms"] = {"lf_parse_file": statistics.median(parse_ms(j.LfParsedFrame, f, a.reps) for f in files[:8]),
                            "parse_file": statistics.median(parse_ms(j.ParsedFrame, f, 3) for f in files[:8])}
    if a.cpu_only:
        print(json.dumps(res))
        return
    import torch
    res["card"] = card()
    ctx = j.JxgContext(0)
    frames = [j.LfParsedFrame(f) for f in files]
    outs = [torch.empty((fr.height, fr.width, 3), dtype=torch.uint8, device="cuda:0") for fr in frames]
    b = j.ModularBatch(ctx)
    try:
        for fr, t in zip(frames, outs):
            b.add_lf(fr, t.data_ptr(), fr.width * 3, 0, True)
        b.run()
        b.wait()
        st = torch.cuda.Stream()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for i in range(a.warmup + a.reps):
            with torch.cuda.stream(st):
                ev0.record(st)
                b.rerun_device(st.cuda_stream)
                ev1.record(st)
            ev1.synchronize()
            if i >= a.warmup:
                times.append(ev0.elapsed_time(ev1))
        b.wait()
        stats = b.stats()
    finally:
        b.close()
        ctx.close()
    ms = statistics.median(times)
    res["device_ms_per_batch"] = ms
    res["thumbnails_per_s"] = a.frames / (ms * 1e-3)
    res["decode_ms_first_run"] = stats["decode_ms"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
