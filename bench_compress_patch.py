#!/usr/bin/env python3
"""bench_compress_patch.py -- delta compression against a reference (B200Z_FLAG_DICT_LONG, libzstd's --patch-from).

    python bench_compress_patch.py [--steps K] [--warmup W] [--skip-cpu] [--total BYTES]

Workload: bench_compress_long.py's "versions" at --total bytes (1 GiB by default): a base of total / 16 bytes of datagen text is the
reference, a raw-content dictionary; its 15 copies, each with about 1 % of its bytes replaced by seeded random runs of 1-32 bytes,
are 15 frames of one submission against it, device-resident, at window_log 27.
Rows, for Fastest, LAZY and OPT:
  patch      with the flag: the ratio (the copies' bytes over the frames'), the call's time (CUDA events around the call, median of
             the steps) and each kernel's milliseconds from one torch.profiler run;
  dict_only  the same frames against the same dictionary without the flag (long matches inside each frame only);
and once: the dictionary's first-use anchor build (a fresh dictionary's first flagged call on one 128 KiB frame, less the same
call once built, wall clock, median of the steps), libzstd 1.5.5 one thread with ZSTD_CCtx_refPrefix(reference),
enableLongDistanceMatching and windowLog 27 at levels 1 and 3 (one frame per copy), and decode_all's time for the 15 Fastest frames
with the reference forced.  Every output, libzstd's included, is decoded on the GPU and must equal its input.  Prints one JSON line
with the card's name and power limit.  Nothing is written to the tree.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_compress import card_info  # noqa: E402
from bench_compress_long import kernel_ms, versions  # noqa: E402

WL = 27


def gpu_rows(pkg, ctx, d_in, io, R, level, dict_long, args):
    """The 15-frame call against R at window_log 27: time, kernels, ratio; every frame decoded on the GPU with R forced."""
    import torch
    cap = int(io["dst_off"][-1] + io["dst_cap"][-1])
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    call = lambda: pkg.compress_frames(ctx, d_in, io, d_out, level, True, R, False, WL, dict_long)  # noqa: E731
    res = call()
    parts = [d_out[int(o):int(o) + int(r["dst_size"])] for o, r in zip(io["dst_off"], res)]
    check(pkg, ctx, parts, d_in, R)
    frames = torch.cat(parts)
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
    size = int(res["dst_size"].sum())
    return {"ms": round(float(np.median(times)), 2), "ms_min_max": [round(min(times), 2), round(max(times), 2)],
            "ratio": round(d_in.numel() / size, 4), "bytes": size, "kernel_ms": kernel_ms(call)}, frames


def check(pkg, ctx, parts, d_in, R):
    """Each frame of `parts` decoded on the GPU (decode_all, the reference forced) equals its 1/15 of d_in."""
    import torch
    n = d_in.numel() // len(parts)
    back = torch.empty(n + 64, dtype=torch.uint8, device="cuda")
    for k, f in enumerate(parts):
        r, _ = pkg.decode_all(ctx, f, back, forced_dict=R, max_window_size=1 << WL)
        assert r["status"] == 0 and torch.equal(back[:n], d_in[k * n:(k + 1) * n]), f"frame {k}: GPU decode differs from the input ({r})"


def decode_ms(pkg, ctx, frames, total, R, args):
    import torch
    back = torch.empty(total + 64, dtype=torch.uint8, device="cuda")
    for _ in range(max(1, args.warmup)):
        pkg.decode_all(ctx, frames, back, forced_dict=R, max_window_size=1 << WL)
    times = []
    for _ in range(args.steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pkg.decode_all(ctx, frames, back, forced_dict=R, max_window_size=1 << WL)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(times)), 2)


def anchor_build_ms(pkg, ctx, base, one, args):
    """A fresh dictionary's first flagged call on one frame less the same call with its anchors built (ms, median of the steps)."""
    import torch
    io = np.array([(0, len(one), 0, pkg.compress_bound(len(one)))], dtype=pkg.binding.COMPRESS_IO_DTYPE)
    out = np.zeros(int(io["dst_cap"][0]), dtype=np.uint8)
    first, later = [], []
    for _ in range(args.steps):
        R = pkg.Dictionary.raw_content(ctx, 0, base)
        pkg.compress_frames(ctx, one, io, out, pkg.FASTEST, True, R, False, WL, False)   # the match table, not timed
        for t in (first, later):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pkg.compress_frames(ctx, one, io, out, pkg.FASTEST, True, R, False, WL, True)
            t.append((time.perf_counter() - t0) * 1e3)
        del R
    return {"first_call_ms": round(float(np.median(first)), 2), "later_call_ms": round(float(np.median(later)), 2),
            "anchor_build_ms": round(float(np.median(first) - np.median(later)), 2)}


def libzstd_patch(pkg, ctx, base, copies, level, R):
    """libzstd one thread, one frame per copy, ZSTD_CCtx_refPrefix(base) before each, long-distance matching, windowLog 27:
    (ratio, seconds); the frames are decoded on the GPU with the reference forced."""
    import torch
    import datagen
    import zmatrix
    z = datagen.zstd()
    z.ZSTD_CCtx_refPrefix.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    z.ZSTD_CCtx_refPrefix.restype = C.c_size_t
    z.ZSTD_compress2.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    z.ZSTD_compress2.restype = C.c_size_t
    z.ZSTD_compressBound.argtypes = [C.c_size_t]
    z.ZSTD_compressBound.restype = C.c_size_t
    z.ZSTD_isError.argtypes = [C.c_size_t]
    z.ZSTD_isError.restype = C.c_uint
    cctx = zmatrix._cctx({"compressionLevel": level, "enableLongDistanceMatching": 1, "windowLog": WL})
    out, dt = [], 0.0
    try:
        for c in copies:
            cap = z.ZSTD_compressBound(len(c))
            dst = np.empty(cap, dtype=np.uint8)
            t0 = time.perf_counter()
            assert not z.ZSTD_isError(z.ZSTD_CCtx_refPrefix(cctx, base.ctypes.data, len(base)))   # a prefix holds for one frame
            n = z.ZSTD_compress2(cctx, dst.ctypes.data, cap, c.ctypes.data, len(c))
            dt += time.perf_counter() - t0
            assert not z.ZSTD_isError(n)
            out.append(dst[:n])
    finally:
        z.ZSTD_freeCCtx(cctx)
    check(pkg, ctx, [torch.from_numpy(f).cuda() for f in out], torch.from_numpy(np.concatenate(copies)).cuda(), R)
    return {"ratio": round(sum(map(len, copies)) / sum(map(len, out)), 4), "s": round(dt, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--total", type=int, default=1 << 30)
    ap.add_argument("--skip-cpu", action="store_true")
    args = ap.parse_args()
    import torch
    import _pkg
    if not torch.cuda.is_available():
        raise SystemExit("bench_compress_patch.py needs a CUDA device: the product path has no CPU fallback")
    pkg = _pkg.load()
    ctx = pkg.Context(0)
    plain = versions(args.total)
    n = args.total // 16
    base, copies = plain[:n], [plain[n * (k + 1):n * (k + 2)] for k in range(15)]
    line = {"metric": "compress_patch", "card": card_info(), "reference_bytes": n, "frames": 15, "frame_bytes": n, "window_log": WL,
            "rows": {}}
    R = pkg.Dictionary.raw_content(ctx, 0, base.tobytes())
    d_in = torch.from_numpy(plain[n:]).cuda()
    io = np.zeros(15, dtype=pkg.binding.COMPRESS_IO_DTYPE)
    cap = pkg.compress_bound(n, R)
    for k in range(15):
        io[k] = (k * n, n, k * cap, cap)
    for lname, level in (("fastest", pkg.FASTEST), ("lazy", pkg.LAZY), ("opt", pkg.OPT)):
        for mode, flag in (("patch", True), ("dict_only", False)):
            line["rows"][f"{lname}_{mode}"], frames = gpu_rows(pkg, ctx, d_in, io, R, level, flag, args)
            print(f"{lname}_{mode}: {line['rows'][f'{lname}_{mode}']}", file=sys.stderr, flush=True)   # progress
            if lname == "fastest" and flag:
                line["rows"]["decode_all_fastest_patch_ms"] = decode_ms(pkg, ctx, frames, d_in.numel(), R, args)
            del frames
    line["rows"]["first_use"] = anchor_build_ms(pkg, ctx, base.tobytes(), copies[0][:131072].tobytes(), args)
    if not args.skip_cpu:
        for lv in (1, 3):
            line["rows"][f"libzstd_l{lv}_refprefix_ldm_w27"] = libzstd_patch(pkg, ctx, base, copies, lv, R)
    del R, d_in
    ctx.close()
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())
