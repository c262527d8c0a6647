#!/usr/bin/env python3
"""bench_compress.py -- input GB/s of the batch compressor (b200z_compress_frames_batch, ruzstd's Fastest level, checksum on).

    python bench_compress.py [--steps K] [--warmup W] [--skip-cpu] [--level fastest|lazy|opt|ultra] [--window-log N]

The workload is the C2b plaintext (1 GiB of enwik9-shaped text, datagen.c2_text_plain), device-resident, in two shapes:
8192 frames of 128 KiB and one 1 GiB frame (C2a's plaintext shape, where the content checksum is four serial chains).
Prints one JSON line: per shape the input GB/s (CUDA events around the call, median of the steps), the ratio, each kernel's
milliseconds, (input + output bytes) / t against the HBM peak, the card's name and power limit, and `cpu_baseline`:
libzstd 1.5.5 level 1 on the same 128 KiB pieces, one thread and all host threads.  --level lazy measures the LAZY extension
level instead, and adds libzstd level 3 to the baseline; --level opt measures the OPT extension level and adds libzstd levels 3
and 16 (btopt, the price-based parse).  --level ultra measures the ULTRA extension level on the one-frame shape at --window-log
(23 by default) against OPT at the same window_log, the two alternated step by step in one run; its far-stage kernels' times come
from torch.profiler, and the baselines are libzstd levels 3, 16 and 19 at that window_log (one frame per 64 MiB piece, the pieces
on all host threads).  Nothing is written to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (measured_peak, host_threads)

GB = 1e9


def card_info():
    """Name and enforced power limit of GPU 0 (read-only NVML queries)."""
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        import pynvml
        pynvml.nvmlInit()
        info["power_limit_W"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        try:
            out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], text=True)
            info["power_limit_W"] = float(out.strip().splitlines()[0])
        except Exception as e:
            info["power_limit_W"] = f"unknown ({str(e)[:60]})"
    return info


def libzstd_compress_baseline(datas, level=1):
    """libzstd 1.5.5 at `level` (one frame per piece): one thread on the first 64 pieces, and all host threads on all of them."""
    import datagen as G
    from concurrent.futures import ThreadPoolExecutor
    sub = datas[:64]
    t0 = time.perf_counter()
    n1 = sum(len(G.compress(d, level=level)) for d in sub)
    one = sum(len(d) for d in sub) / (time.perf_counter() - t0) / GB
    threads = bench.host_threads()
    with ThreadPoolExecutor(max_workers=threads) as ex:
        t0 = time.perf_counter()
        sizes = list(ex.map(lambda d: len(G.compress(d, level=level)), datas))
        dt = time.perf_counter() - t0
    total = sum(len(d) for d in datas)
    return {"kind": f"libzstd 1.5.5 level {level}", "one_core_GBps": one, "one_core_ratio": sum(len(d) for d in sub) / n1,
            "all_cores_GBps": total / dt / GB, "cores": threads, "ratio": total / sum(sizes)}


def run_compress(args):
    """b200z_compress_frames_batch at the Fastest (or LAZY, or OPT) level on the 1 GiB C2b plaintext, device-resident, in two shapes:
    8192 frames of 128 KiB (C2b) and one 1 GiB frame (C2a's plaintext shape).  Each output is first decoded on the GPU and must
    equal the input; then the call is timed with CUDA events after warm-up, and one more run with a CUDA event between kernels
    gives each kernel's time."""
    import torch
    import _pkg
    import datagen
    if not torch.cuda.is_available():
        raise SystemExit("bench_compress.py needs a CUDA device: the product path has no CPU fallback")
    pkg = _pkg.load()
    ctx = pkg.Context(0)
    total = args.c2a_bytes
    plain = datagen.c2_text_plain(total)
    d_in = torch.from_numpy(plain).cuda()
    peak, peak_src = bench.measured_peak()
    level, name = {"fastest": (pkg.FASTEST, "Fastest"), "lazy": (pkg.LAZY, "LAZY"), "opt": (pkg.OPT, "OPT")}[args.level]
    line = {"metric": "compress_GBps", "unit": "GB/s", "level": name, "checksum": True, "card": card_info(), "input_bytes": total, "shapes": {}}
    for shape, frame_bytes in (("c2b", args.frame_bytes), ("c2a", total)):
        nfr = total // frame_bytes
        io = np.zeros(nfr, dtype=pkg.binding.COMPRESS_IO_DTYPE)
        cap = pkg.compress_bound(frame_bytes)
        for i in range(nfr):
            io[i] = (i * frame_bytes, frame_bytes, i * cap, cap)
        d_out = torch.empty(nfr * cap, dtype=torch.uint8, device="cuda")
        res = pkg.compress_frames(ctx, d_in, io, d_out, level)
        assert (res["status"] == 0).all()
        dio = np.zeros(nfr, dtype=pkg.binding.FRAME_IO_DTYPE)
        dio["src_off"], dio["src_size"], dio["out_off"], dio["out_cap"] = io["dst_off"], res["dst_size"], io["src_off"], frame_bytes
        back = torch.empty(total + 16, dtype=torch.uint8, device="cuda")
        dres = pkg.decode_frames(ctx, d_out, dio, back)
        assert (dres["status"] == 0).all() and torch.equal(back[:total], d_in), f"{shape}: GPU decode of the compressed frames differs from the input"
        del back
        for _ in range(args.warmup):
            pkg.compress_frames(ctx, d_in, io, d_out, level)
        stream = torch.cuda.ExternalStream(ctx.stream())
        times = []
        for _ in range(args.steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            pkg.compress_frames(ctx, d_in, io, d_out, level)
            b.record(stream)
            b.synchronize()
            times.append(a.elapsed_time(b) / 1e3)
        ctx.set_flags(pkg.binding.FLAG_PROFILE)
        pkg.compress_frames(ctx, d_in, io, d_out, level)
        prof = pkg.compress_profile(ctx)
        ctx.set_flags(0)
        t = float(np.median(times))
        out_bytes = int(res["dst_size"].sum())
        line["shapes"][shape] = {"frames": nfr, "frame_bytes": frame_bytes, "value": total / t / GB, "ms": t * 1e3,
                                 "ms_min_max": [min(times) * 1e3, max(times) * 1e3], "ratio": total / out_bytes, "output_bytes": out_bytes,
                                 "kernel_ms": prof, "roofline": {"bytes_per_call": total + out_bytes, "peak_GBps": peak, "peak_source": peak_src,
                                                                 "fraction": (total + out_bytes) / t / GB / peak},
                                 "raw_blocks": int(res["raw_blocks"].sum()), "rle_blocks": int(res["rle_blocks"].sum()), "blocks": int(res["blocks"].sum())}
        del d_out
    line["value"], line["ratio"] = line["shapes"]["c2b"]["value"], line["shapes"]["c2b"]["ratio"]
    if not args.skip_cpu:
        pieces = [plain[i:i + args.frame_bytes] for i in range(0, total, args.frame_bytes)]
        line["cpu_baseline"] = libzstd_compress_baseline(pieces)
        if args.level in ("lazy", "opt"):
            line["cpu_baseline_level3"] = libzstd_compress_baseline(pieces, 3)
        if args.level == "opt":
            line["cpu_baseline_level16"] = libzstd_compress_baseline(pieces, 16)
    ctx.close()
    print(json.dumps(line))


FAR_KERNELS = ("k_fkey", "k_lhist", "k_lscan", "k_lscatter", "k_fstart", "k_copt", "k_lanchor", "k_lcand", "k_lblock")


def libzstd_window_baseline(plain, level, window_log, piece=64 << 20):
    """libzstd 1.5.5 at `level` and window_log, one frame per `piece` bytes, the pieces on all host threads."""
    import datagen as G
    from concurrent.futures import ThreadPoolExecutor
    pieces = [plain[i:i + piece].tobytes() for i in range(0, len(plain), piece)]
    with ThreadPoolExecutor(max_workers=bench.host_threads()) as ex:
        t0 = time.perf_counter()
        sizes = list(ex.map(lambda d: len(G.compress(d, level=level, window_log=window_log)), pieces))
        dt = time.perf_counter() - t0
    return {"kind": f"libzstd 1.5.5 level {level}, window_log {window_log}, {piece >> 20} MiB frames", "all_cores_GBps": len(plain) / dt / GB,
            "cores": bench.host_threads(), "ratio": len(plain) / sum(sizes)}


def run_ultra(args):
    """ULTRA and OPT on one frame of the C2b plaintext at --window-log, alternated; each output decodes on the GPU to the input."""
    import torch
    import _pkg
    import datagen
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("bench_compress.py needs a CUDA device: the product path has no CPU fallback")
    pkg = _pkg.load()
    ctx = pkg.Context(0)
    total, wl = args.c2a_bytes, args.window_log
    plain = datagen.c2_text_plain(total)
    d_in = torch.from_numpy(plain).cuda()
    io = np.zeros(1, dtype=pkg.binding.COMPRESS_IO_DTYPE)
    cap = pkg.compress_bound(total)
    io[0] = (0, total, 0, cap)
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    line = {"metric": "compress_GBps", "unit": "GB/s", "level": "ULTRA", "window_log": wl, "checksum": True, "card": card_info(),
            "input_bytes": total, "frames": 1, "levels": {}}
    levels = (("ULTRA", pkg.ULTRA), ("OPT", pkg.OPT))
    for name, level in levels:
        res = pkg.compress_frames(ctx, d_in, io, d_out, level, window_log=wl)
        assert (res["status"] == 0).all()
        dio = np.zeros(1, dtype=pkg.binding.FRAME_IO_DTYPE)
        dio["src_off"], dio["src_size"], dio["out_off"], dio["out_cap"] = 0, res["dst_size"], 0, total
        back = torch.empty(total + 16, dtype=torch.uint8, device="cuda")
        dres = pkg.decode_frames(ctx, d_out, dio, back)
        assert (dres["status"] == 0).all() and torch.equal(back[:total], d_in), f"{name}: GPU decode differs from the input"
        del back
        line["levels"][name] = {"ratio": total / int(res["dst_size"][0]), "output_bytes": int(res["dst_size"][0]), "times": []}
        for _ in range(args.warmup):
            pkg.compress_frames(ctx, d_in, io, d_out, level, window_log=wl)
    stream = torch.cuda.ExternalStream(ctx.stream())
    for _ in range(args.steps):
        for name, level in levels:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            pkg.compress_frames(ctx, d_in, io, d_out, level, window_log=wl)
            b.record(stream)
            b.synchronize()
            line["levels"][name]["times"].append(a.elapsed_time(b))
    for name, level in levels:
        r = line["levels"][name]
        t = float(np.median(r["times"]))
        r.update({"ms": t, "ms_min_max": [min(r["times"]), max(r["times"])], "value": total / (t / 1e3) / GB})
        ctx.set_flags(pkg.binding.FLAG_PROFILE)
        pkg.compress_frames(ctx, d_in, io, d_out, level, window_log=wl)
        r["stage_ms"] = pkg.compress_profile(ctx)
        ctx.set_flags(0)
        with profile(activities=[ProfilerActivity.CUDA]) as pr:
            pkg.compress_frames(ctx, d_in, io, d_out, level, window_log=wl)
            torch.cuda.synchronize()
        ms = {}
        for ev in pr.key_averages():
            k = next((k for k in FAR_KERNELS if k in ev.key), None)
            if k:
                ms[k] = ms.get(k, 0.0) + ev.device_time_total / 1e3
        r["kernel_ms_profiler"] = ms
    line["value"], line["ratio"] = line["levels"]["ULTRA"]["value"], line["levels"]["ULTRA"]["ratio"]
    if not args.skip_cpu:
        line["cpu_baselines"] = [libzstd_window_baseline(plain, lv, wl) for lv in (3, 16, 19)]
    ctx.close()
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frame-bytes", type=int, default=131072)
    ap.add_argument("--c2a-bytes", type=int, default=1 << 30, help="total plaintext bytes (both shapes)")
    ap.add_argument("--skip-cpu", action="store_true")
    ap.add_argument("--level", choices=("fastest", "lazy", "opt", "ultra"), default="fastest")
    ap.add_argument("--window-log", type=int, default=23, help="--level ultra: the window_log of both levels and the baselines")
    args = ap.parse_args()
    (run_ultra if args.level == "ultra" else run_compress)(args)
    return 0


if __name__ == "__main__":
    sys.exit(main())
