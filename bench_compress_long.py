#!/usr/bin/env python3
"""bench_compress_long.py -- the compressor's long-distance matches (window_log > 17) on large inputs whose redundancy lies megabytes apart.

    python bench_compress_long.py [--steps K] [--warmup W] [--skip-cpu] [--total BYTES]

Workloads (--total bytes each, 1 GiB by default):
  (a) the C2b plaintext (datagen.c2_text_plain) as one frame, at window_log 17 and 27;
  (b) "versions": a base of 1/16 of the total of datagen text and 15 copies of it, each with about 1 % of its bytes replaced by
      seeded random runs of 1-32 bytes, as one frame at window_log 17 and 27;
  (c) (b) through FrameCompressor, host to host, at the default chunk (64 MiB), at window_log 17 and 27.
For Fastest and LAZY: the call's time (CUDA events around the device-resident call, median of the steps; wall clock for (c)),
each kernel's milliseconds from one torch.profiler run (the long-match kernels included), and the ratio.  libzstd 1.5.5 at levels 1
and 3 with enableLongDistanceMatching and windowLog 27, one thread, on (a) and (b): ratio and time.  decode_all's time for (b)'s
frame at 27.  Every output is decoded on the GPU and must equal its input.  Prints one JSON line with the card's name and power
limit.  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_compress import card_info  # noqa: E402

LDM_KERNELS = ("k_lanchor", "k_lscan", "k_lhist", "k_lscatter", "k_lcand", "k_lblock")


def versions(total, seed=0x10A6):
    """A base of total / 16 bytes of datagen text, then 15 copies with about 1 % of their bytes replaced by random runs of 1-32."""
    import datagen
    n = total // 16
    base = datagen.gen_text(n, seed)
    rng = np.random.default_rng(seed)
    out = [base]
    for _ in range(15):
        v = base.copy()
        runs = int(0.01 * n / 16.5)
        at = rng.integers(0, n - 32, runs)
        ln = rng.integers(1, 33, runs)
        for a, k in zip(at.tolist(), ln.tolist()):
            v[a:a + k] = rng.integers(0, 256, k, dtype=np.uint8)
        out.append(v)
    return np.concatenate(out)


def kernel_ms(fn):
    """{kernel name: ms} of one call of fn under torch.profiler (CUDA activity), summed per name."""
    import re
    import torch
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        m = re.search(r"b200z::(k_\w+)", e.key)
        if m:
            out[m.group(1)] = out.get(m.group(1), 0.0) + e.device_time_total / 1e3
    return {k: round(v, 3) for k, v in sorted(out.items())}


def libzstd_ldm(plain, level):
    """libzstd one thread at `level` with long-distance matching and windowLog 27: (ratio, seconds)."""
    import datagen
    import zmatrix
    z = datagen.zstd()
    cap = z.ZSTD_compressBound(len(plain))
    dst = np.empty(cap, dtype=np.uint8)
    cctx = zmatrix._cctx({"compressionLevel": level, "enableLongDistanceMatching": 1, "windowLog": 27})
    try:
        t0 = time.perf_counter()
        n = z.ZSTD_compress2(cctx, dst.ctypes.data, cap, plain.ctypes.data, len(plain))
        dt = time.perf_counter() - t0
    finally:
        z.ZSTD_freeCCtx(cctx)
    assert not z.ZSTD_isError(n)
    return {"ratio": round(len(plain) / n, 4), "s": round(dt, 3)}


def one_frame(pkg, ctx, d_in, level, window_log, args):
    """The device-resident one-frame call: time, kernels, ratio; decoded on the GPU against the input."""
    import torch
    total = d_in.numel()
    cap = pkg.compress_bound(total)
    io = np.array([(0, total, 0, cap)], dtype=pkg.binding.COMPRESS_IO_DTYPE)
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    call = lambda: pkg.compress_frames(ctx, d_in, io, d_out, level, True, None, False, window_log)  # noqa: E731
    res = call()
    size = int(res[0]["dst_size"])
    back = torch.empty(total + 64, dtype=torch.uint8, device="cuda")
    r = pkg.decode_all(ctx, d_out[:size], back)
    assert torch.equal(back[:total], d_in), f"window_log {window_log}: GPU decode differs from the input ({r})"
    del back
    for _ in range(args.warmup):
        call()
    stream = torch.cuda.ExternalStream(ctx.stream())
    times = []
    for _ in range(args.steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        call()
        b.record(stream)
        b.synchronize()
        times.append(a.elapsed_time(b))
    ks = kernel_ms(call)
    ldm = sum(v for k, v in ks.items() if k in LDM_KERNELS)
    out = {"ms": round(float(np.median(times)), 2), "ms_min_max": [round(min(times), 2), round(max(times), 2)], "ratio": round(total / size, 4),
           "bytes": size, "kernel_ms": ks, "ldm_ms": round(ldm, 3)}
    if "k_cmatch" in ks:
        out["ldm_share_of_k_cmatch"] = round(ldm / ks["k_cmatch"], 4)
    return out, d_out[:size].clone()


def decode_ms(pkg, ctx, frame, total, args):
    import torch
    back = torch.empty(total + 64, dtype=torch.uint8, device="cuda")
    for _ in range(max(1, args.warmup)):
        pkg.decode_all(ctx, frame, back)
    times = []
    for _ in range(args.steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pkg.decode_all(ctx, frame, back)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(times)), 2)


def stream_run(pkg, ctx, plain, level, window_log):
    """FrameCompressor host to host: (seconds, ratio); the frame is decoded by libzstd against the input."""
    import datagen
    fc = pkg.FrameCompressor(ctx, level, True, window_log)
    src = memoryview(plain)
    out = bytearray()
    fc.set_source(src.tobytes())
    fc.set_drain(out)
    t0 = time.perf_counter()
    r = fc.compress()
    dt = time.perf_counter() - t0
    assert r["status"] == 0
    assert datagen.decompress(bytes(out), len(plain), window_log_max=27) == bytes(plain)
    return {"s": round(dt, 3), "ratio": round(len(plain) / len(out), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--total", type=int, default=1 << 30)
    ap.add_argument("--skip-cpu", action="store_true")
    args = ap.parse_args()
    import torch
    import _pkg
    import datagen
    if not torch.cuda.is_available():
        raise SystemExit("bench_compress_long.py needs a CUDA device: the product path has no CPU fallback")
    pkg = _pkg.load()
    ctx = pkg.Context(0)
    line = {"metric": "compress_long", "card": card_info(), "input_bytes": args.total, "workloads": {}}
    inputs = {"a_c2b_text": datagen.c2_text_plain(args.total), "b_versions": versions(args.total)}
    for name, plain in inputs.items():
        d_in = torch.from_numpy(plain).cuda()
        w = line["workloads"][name] = {}
        for lname, level in (("fastest", pkg.FASTEST), ("lazy", pkg.LAZY)):
            for wl in (17, 27):
                w[f"{lname}_w{wl}"], frame = one_frame(pkg, ctx, d_in, level, wl, args)
                if name == "b_versions" and lname == "fastest":
                    w[f"{lname}_w{wl}"]["decode_all_ms"] = decode_ms(pkg, ctx, frame, len(plain), args)
                del frame
        if not args.skip_cpu:
            for lv in (1, 3):
                w[f"libzstd_l{lv}_ldm_w27"] = libzstd_ldm(plain, lv)
        if name == "b_versions":
            s = line["workloads"]["c_versions_stream"] = {}
            for lname, level in (("fastest", pkg.FASTEST), ("lazy", pkg.LAZY)):
                for wl in (17, 27):
                    s[f"{lname}_w{wl}"] = stream_run(pkg, ctx, plain, level, wl)
        del d_in
    ctx.close()
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())
