#!/usr/bin/env python3
"""bench_seekable.py -- seekable archives on the GPU: writing (b200z_compress_seekable) and random reads (b200z_seekable_read_ranges).

    python bench_seekable.py [--steps K] [--warmup W] [--total BYTES] [--frame-bytes N] [--ranges N]

The workload is the C2b plaintext (1 GiB of enwik9-shaped text, datagen.c2_text_plain), device-resident, at Fastest with checksums.
Prints one JSON line with the card's name and power limit and, timed with CUDA events (median of the steps):
  compress: compress_seekable at --frame-bytes against compress_frames on the same pieces, alternated step by step; GB/s of input
            and the ratio of each (the archive's against the frames' sum);
  random:   batches of --ranges ranges of 4-64 KiB at seeded random offsets from the device archive into device memory, each batch
            new: ms per batch, requested GB/s (bytes asked for) and decoded GB/s (plaintext of the frames touched);
  one_4k:   one 4 KiB read, ms;
  decode_all: the whole archive through decode_all (tier 1c), GB/s of plaintext.
Every result is checked against the input first.  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_compress import card_info  # noqa: E402

GB = 1e9


def random_batch(pkg, total, n, rng):
    """n ranges of 4-64 KiB at random offsets, output slots back to back"""
    b = np.zeros(n, dtype=pkg.binding.RANGE_DTYPE)
    b["length"] = rng.integers(4096, 65537, n)
    b["offset"] = (rng.random(n) * (total - b["length"] + 1)).astype(np.uint64)
    b["out_off"] = np.concatenate(([0], np.cumsum(b["length"])[:-1]))
    return b


def decoded_bytes(starts, b):
    """plaintext bytes of the distinct frames the ranges touch (each decoded once)"""
    lo = np.searchsorted(starts, b["offset"].astype(np.int64), side="right") - 1
    hi = np.searchsorted(starts, (b["offset"] + b["length"]).astype(np.int64), side="left")
    touched = np.unique(np.concatenate([np.arange(x, y) for x, y in zip(lo, hi)]))
    return int((starts[touched + 1] - starts[touched]).sum())


def timed(stream, fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--total", type=int, default=1 << 30)
    ap.add_argument("--frame-bytes", type=int, default=131072)
    ap.add_argument("--ranges", type=int, default=4096)
    args = ap.parse_args()
    import torch
    import _pkg
    import datagen
    if not torch.cuda.is_available():
        raise SystemExit("bench_seekable.py needs a CUDA device: the product path has no CPU fallback")
    pkg = _pkg.load()
    ctx = pkg.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream())
    total, fs = args.total, args.frame_bytes
    plain = datagen.c2_text_plain(total)
    d_in = torch.from_numpy(plain).cuda()
    line = {"metric": "seekable", "card": card_info(), "input_bytes": total, "frame_bytes": fs, "level": "Fastest", "checksum": True}

    # ---- writing, alternated with compress_frames on the same pieces
    cap = pkg.seekable_bound(total, fs, True)
    d_arch = torch.empty(cap, dtype=torch.uint8, device="cuda")
    nfr = -(-total // fs)
    io = np.zeros(nfr, dtype=pkg.binding.COMPRESS_IO_DTYPE)
    fcap = pkg.compress_bound(fs)
    for i in range(nfr):
        io[i] = (i * fs, min(fs, total - i * fs), i * fcap, fcap)
    d_frames = torch.empty(nfr * fcap, dtype=torch.uint8, device="cuda")
    n = pkg.compress_seekable(ctx, d_in, d_arch, fs)
    res = pkg.compress_frames(ctx, d_in, io, d_frames)
    back = torch.empty(total + 64, dtype=torch.uint8, device="cuda")
    s, _ = pkg.decode_all(ctx, d_arch[:n], back)
    assert s["status"] == 0 and s["written"] == total and torch.equal(back[:total], d_in), "the archive does not decode to the input"
    for _ in range(args.warmup):
        pkg.compress_seekable(ctx, d_in, d_arch, fs)
        pkg.compress_frames(ctx, d_in, io, d_frames)
    ts, tf = [], []
    for _ in range(args.steps):
        ts.append(timed(stream, lambda: pkg.compress_seekable(ctx, d_in, d_arch, fs)))
        tf.append(timed(stream, lambda: pkg.compress_frames(ctx, d_in, io, d_frames)))
    t_s, t_f = float(np.median(ts)), float(np.median(tf))
    line["compress"] = {"seekable_GBps": total / t_s / GB, "seekable_ms": t_s * 1e3, "seekable_ratio": total / n, "archive_bytes": n,
                        "frames_GBps": total / t_f / GB, "frames_ms": t_f * 1e3, "frames_ratio": total / int(res["dst_size"].sum()),
                        "seekable_over_frames_time": t_s / t_f}
    del d_frames

    # ---- random reads from the device archive into device memory
    arch = d_arch[:n]
    rng = np.random.default_rng(0x5EEC)
    with pkg.SeekableArchive(ctx, arch) as a:
        fr = a.frames
        starts = np.append(fr["d_off"], total).astype(np.int64)
        batches = [random_batch(pkg, total, args.ranges, rng) for _ in range(args.warmup + args.steps)]
        out = torch.empty(max(int(b["out_off"][-1] + b["length"][-1]) for b in batches) + 16, dtype=torch.uint8, device="cuda")
        check = a.read_ranges(batches[0], out)
        assert (check["status"] == 0).all()
        host_out = out.cpu().numpy()
        for off, ln, oo in batches[0][:256]:
            assert (host_out[oo:oo + ln] == plain[off:off + ln]).all(), "a range differs from the input"
        times = []
        for i, b in enumerate(batches):
            t = timed(stream, lambda: a.read_ranges(b, out))
            if i >= args.warmup:
                times.append(t)
        t_r = float(np.median(times))
        req = float(np.mean([int(b["length"].sum()) for b in batches[args.warmup:]]))
        dec = float(np.mean([decoded_bytes(starts, b) for b in batches[args.warmup:]]))
        line["random"] = {"ranges_per_batch": args.ranges, "range_bytes": [4096, 65536], "ms_per_batch": t_r * 1e3,
                          "ms_min_max": [min(times) * 1e3, max(times) * 1e3], "requested_GBps": req / t_r / GB, "decoded_GBps": dec / t_r / GB,
                          "requested_bytes": req, "decoded_bytes": dec}
        one = []
        for i in range(args.warmup + args.steps):
            off = int(rng.integers(0, total - 4096))
            t = timed(stream, lambda: a.read_ranges([(off, 4096, 0)], out))
            if i >= args.warmup:
                one.append(t)
        assert (out[:4096].cpu().numpy() == plain[off:off + 4096]).all()
        line["one_4k"] = {"ms": float(np.median(one)) * 1e3, "ms_min_max": [min(one) * 1e3, max(one) * 1e3]}

    # ---- the whole archive through decode_all
    td = []
    for i in range(args.warmup + args.steps):
        t = timed(stream, lambda: pkg.decode_all(ctx, arch, back))
        if i >= args.warmup:
            td.append(t)
    t_d = float(np.median(td))
    line["decode_all"] = {"GBps": total / t_d / GB, "ms": t_d * 1e3}
    line["value"] = line["random"]["requested_GBps"]
    line["unit"] = "GB/s requested, random reads"
    ctx.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
