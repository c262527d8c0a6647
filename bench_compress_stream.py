#!/usr/bin/env python3
"""bench_compress_stream.py -- input GB/s of the stream compressor (FrameCompressor.compress, b200z_frame_compressor) against
the batch compressor, host memory to host memory, Fastest level, checksum on.

    python bench_compress_stream.py [--steps K] [--bytes N] [--skip-cpu]

Workload: the C2b plaintext (1 GiB of enwik9-shaped text, datagen.c2_text_plain) in host memory.  Arms, alternated step by step
in one run, wall time around each call:
  stream       FrameCompressor.compress at the default chunk; its read and write callbacks memmove from the plaintext and into a
               preallocated host buffer
  batch_1      compress_frames with one frame of the whole input, host to host
  batch_8192   compress_frames with 128 KiB frames (8192 for 1 GiB), host to host
  libzstd_1    libzstd 1.5.5 level 1, one thread, one frame
  host_only    the stream arm's host work alone, on the same thread: the read callback into a pinned 64 MiB buffer and XXH64 of
               it per chunk, then the write callback of as many bytes as the stream arm wrote (what the stream cannot go below)
Prints one JSON line: per arm the median and min-max GB/s of input and milliseconds, the ratio and the kernel launches per call;
the card's name and power limit; the device memory the stream compressor holds (free device memory before and after its first
call, the kernels loaded beforehand; other processes on the card can disturb it) beside the header's formula; and the device
time of k_cmatch + k_cenc + k_cassemble on the same 8192 blocks, device-resident, checksum off (the stream's kernel work).
Outside the timing, the stream frame's blocks are checked against the one-frame batch frame's (tests/streamframe.py).
Nothing is written to the tree.
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

GB = 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--bytes", type=int, default=1 << 30)
    ap.add_argument("--skip-cpu", action="store_true")
    args = ap.parse_args()
    import torch
    import _pkg
    import datagen
    import streamframe as SF
    from bench_compress import card_info
    if not torch.cuda.is_available():
        raise SystemExit("bench_compress_stream.py needs a CUDA device: the product path has no CPU fallback")
    pkg = _pkg.load()
    B = pkg.binding
    L = pkg.lib()
    ctx = pkg.Context(0)
    total = args.bytes
    plain = datagen.c2_text_plain(total)
    src_addr = plain.ctypes.data

    # ---- (a) the stream compressor over memmove callbacks
    s_out = np.empty(pkg.compress_bound(total), dtype=np.uint8)
    pos = {"r": 0, "w": 0}

    def _read(_u, buf, n):
        k = min(n, total - pos["r"])
        C.memmove(buf, src_addr + pos["r"], k)
        pos["r"] += k
        return k

    def _write(_u, buf, n):
        C.memmove(s_out.ctypes.data + pos["w"], buf, n)
        pos["w"] += n
        return n

    rd, wr = B.READ_FN(_read), B.WRITE_FN(_write)
    fc = pkg.FrameCompressor(ctx)
    s_res = np.zeros(1, dtype=B.COMPRESS_RESULT_DTYPE)

    def stream():
        pos["r"] = pos["w"] = 0
        ctx._chk(L.b200z_frame_compressor_compress(fc.h, rd, None, wr, None, s_res.ctypes.data))
        return int(s_res[0]["dst_size"])

    pkg.compress_to_vec(ctx, plain[:1 << 20])   # load the kernels (and their local memory) before measuring the compressor's buffers
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    stream()
    held = free0 - torch.cuda.mem_get_info(0)[0]
    chunk, blk = 64 << 20, 131072
    staging = 2 * blk + 2 * 12 * 8 * ((blk // 8) // 5 + 1) + 2 * 16   # lit_stage, lits, seq_stage, seqs, info, res per block
    formula = 2 * (blk + chunk + 16) + 2 * (chunk + 3 * (chunk // blk) + 16) + (chunk // blk) * staging

    # ---- (b), (c) the batch compressor, host to host
    def batch_io(frame_bytes):
        nfr = -(-total // frame_bytes)
        io = np.zeros(nfr, dtype=B.COMPRESS_IO_DTYPE)
        off = 0
        for i in range(nfr):
            n = min(frame_bytes, total - i * frame_bytes)
            cap = pkg.compress_bound(n)
            io[i] = (i * frame_bytes, n, off, cap)
            off += cap
        return io, np.empty(off, dtype=np.uint8)

    io1, out1 = batch_io(total)
    io8, out8 = batch_io(131072)

    def batch(io, out):
        res = pkg.compress_frames(ctx, plain, io, out)
        return int(res["dst_size"].sum())

    def libzstd():
        return len(datagen.compress(plain, level=1))

    pinned = torch.empty(chunk, dtype=torch.uint8).pin_memory()
    pin = pinned.data_ptr()

    def host_only():
        pos["r"] = 0
        for off in range(0, total, chunk):
            n = min(chunk, total - off)
            _read(None, pin, n)
            L.b200z_xxh64(pin, n)
        pos["r"] = pos["w"] = 0
        left = sizes.get("stream", total)
        while left:
            n = min(chunk, left)
            _write(None, pin, n)
            left -= n
        return sizes.get("stream", total)

    arms = {"stream": stream, "batch_1": lambda: batch(io1, out1), "batch_8192": lambda: batch(io8, out8), "host_only": host_only}
    if not args.skip_cpu:
        arms["libzstd_1"] = libzstd
    sizes = {}

    # ---- the stream frame against the batch frame, once, outside the timing
    frame = s_out[:stream()].tobytes()
    one = out1[:int(pkg.compress_frames(ctx, plain, io1, out1)[0]["dst_size"])].tobytes()
    _, sb, st = SF.split_frame(frame)
    _, bb, bt = SF.split_frame(one)
    full = sb[:-1] if total % SF.BLOCK == 0 else sb
    blocks_equal = [b[1:] for b in full] == [b[1:] for b in bb] and st == bt and len(sb) == total // SF.BLOCK + 1
    assert blocks_equal, "the stream frame's blocks differ from the batch frame's"
    del frame, one

    for f in arms.values():   # warm-up: first-use allocations
        f()
    times = {k: [] for k in arms}
    launches = {}
    for _ in range(args.steps):
        for k, f in arms.items():
            l0 = ctx.kernel_launches()
            t0 = time.perf_counter()
            sizes[k] = f()
            times[k].append(time.perf_counter() - t0)
            launches[k] = ctx.kernel_launches() - l0
    d_in = torch.from_numpy(plain).cuda()
    d_out = torch.empty(int(io8["dst_cap"].sum()), dtype=torch.uint8, device="cuda")
    ctx.set_flags(B.FLAG_PROFILE)
    pkg.compress_frames(ctx, d_in, io8, d_out, checksum=False)
    prof = pkg.compress_profile(ctx)
    ctx.set_flags(0)
    del d_in, d_out
    out = {}
    for k, ts in times.items():
        t = float(np.median(ts))
        out[k] = {"GBps": total / t / GB, "GBps_min_max": [total / max(ts) / GB, total / min(ts) / GB], "ms": t * 1e3,
                  "ms_min_max": [min(ts) * 1e3, max(ts) * 1e3], "ratio": total / sizes[k], "kernel_launches": launches[k]}
    line = {"metric": "compress_stream_GBps", "unit": "GB/s", "value": out["stream"]["GBps"], "level": "Fastest", "checksum": True,
            "input_bytes": total, "steps": args.steps, "card": card_info(), "arms": out,
            "stream_device_bytes_held": int(held), "stream_device_bytes_formula": int(formula),
            "kernel_ms_8192_blocks_device_resident": {k: v for k, v in prof.items() if k != "k_cxxh64"},
            "stream_blocks_equal_batch": bool(blocks_equal)}
    ctx.close()
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())
