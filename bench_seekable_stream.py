#!/usr/bin/env python3
"""bench_seekable_stream.py -- seekable archives larger than memory: the stream writer (b200z_compress_seekable_stream) and reads
through a positional-read callback (b200z_seekable_open_source).

    python bench_seekable_stream.py [--steps K] [--warmup W] [--total BYTES] [--frame-bytes N] [--ranges N]

The workload is the C2b plaintext (1 GiB of enwik9-shaped text, datagen.c2_text_plain) in host memory, at Fastest with checksums.
Arms alternate step by step in one run; each time is a host clock around a call that ends synchronised.  Prints one JSON line with
the card's name and power limit and, for every arm, the median and the min-max of the steps:
  write: host to host.  stream: compress_seekable_stream through ctypes callbacks that memmove from the input and to the output;
         seekable: compress_seekable on the same host buffers; frame_compressor: FrameCompressor's one frame through the same callbacks
         (the stream compressor, which hashes on the host).  GB/s of input.
  read:  batches of --ranges ranges of 4-64 KiB at seeded random offsets into host memory.  file: the archive in a file (in the page
         cache after the first pass) through SeekableArchive.from_source (os.pread); memory: the same batch on the host archive.
Every result is checked first: the stream archive equals compress_seekable's, and both readers return the input's bytes.  Nothing is
written to the tree (the archive file goes to a temporary directory).
"""
import argparse
import ctypes as C
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_compress import card_info  # noqa: E402
from bench_seekable import random_batch  # noqa: E402

GB = 1e9


class MemIO:
    """A source over one host array and a drain into another, as raw ctypes callbacks that memmove (no Python bytes objects)."""

    def __init__(self, pkg, src, dst):
        self.src, self.dst = src, dst
        self.pos = self.out = 0
        B = pkg.binding

        def _read(_u, buf, n):
            k = min(n, len(self.src) - self.pos)
            C.memmove(buf, self.src.ctypes.data + self.pos, k)
            self.pos += k
            return k

        def _write(_u, buf, n):
            if self.out + n > len(self.dst):
                return -1
            C.memmove(self.dst.ctypes.data + self.out, buf, n)
            self.out += n
            return n
        self.rd, self.wr = B.READ_FN(_read), B.WRITE_FN(_write)

    def reset(self):
        self.pos = self.out = 0


def stats(ts):
    return {"ms": float(np.median(ts)) * 1e3, "ms_min_max": [min(ts) * 1e3, max(ts) * 1e3]}


def clock(fn):
    t = time.perf_counter()
    fn()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--total", type=int, default=1 << 30)
    ap.add_argument("--frame-bytes", type=int, default=131072)
    ap.add_argument("--ranges", type=int, default=4096)
    args = ap.parse_args()
    import torch
    import _pkg
    import datagen
    if not torch.cuda.is_available():
        raise SystemExit("bench_seekable_stream.py needs a CUDA device: the product path has no CPU fallback")
    pkg = _pkg.load()
    B = pkg.binding
    ctx = pkg.Context(0)
    L = ctx.L
    total, fs = args.total, args.frame_bytes
    plain = np.ascontiguousarray(datagen.c2_text_plain(total))
    line = {"metric": "seekable_stream", "card": card_info(), "input_bytes": total, "frame_bytes": fs, "level": "Fastest", "checksum": True,
            "chunk_bytes": int(os.environ.get("B200Z_PIPELINE_CHUNK_BYTES", 64 << 20))}

    # ---- writing, host to host
    cap = pkg.seekable_bound(total, fs, True)
    out_seek = np.empty(cap, dtype=np.uint8)
    out_stream = np.empty(cap, dtype=np.uint8)
    out_frame = np.empty(pkg.compress_bound(total) + 64, dtype=np.uint8)
    io_s, io_f = MemIO(pkg, plain, out_stream), MemIO(pkg, plain, out_frame)
    res = np.zeros(1, dtype=B.SEEKABLE_STREAM_RESULT_DTYPE)
    fc = pkg.FrameCompressor(ctx, pkg.FASTEST, True)
    fres = np.zeros(1, dtype=B.COMPRESS_RESULT_DTYPE)

    def run_stream():
        io_s.reset()
        ctx._chk(L.b200z_compress_seekable_stream(ctx.h, io_s.rd, None, io_s.wr, None, fs, pkg.FASTEST, 1, None, res.ctypes.data))

    def run_seek():
        return pkg.compress_seekable(ctx, plain, out_seek, fs)

    def run_frame():
        io_f.reset()
        ctx._chk(L.b200z_frame_compressor_compress(fc.h, io_f.rd, None, io_f.wr, None, fres.ctypes.data))

    n = run_seek()
    run_stream()
    assert io_s.out == n and np.array_equal(out_stream[:n], out_seek[:n]), "the stream archive differs from compress_seekable's"
    groups = int(res[0]["groups"])
    arms = {"stream": run_stream, "seekable": run_seek, "frame_compressor": run_frame}
    times = {k: [] for k in arms}
    for i in range(args.warmup + args.steps):
        for k, fn in arms.items():
            t = clock(fn)
            if i >= args.warmup:
                times[k].append(t)
    line["write"] = {k: dict(stats(v), GBps=total / float(np.median(v)) / GB) for k, v in times.items()}
    line["write"]["archive_bytes"] = n
    line["write"]["stream_groups"] = groups
    line["write"]["frame_compressor_bytes"] = io_f.out

    # ---- random reads: the archive in a file through from_source, against the host archive
    arch = out_seek[:n]
    tmp = tempfile.mkdtemp(prefix="b200z_seek_")
    try:
        path = os.path.join(tmp, "archive.zst")
        arch.tofile(path)
        rng = np.random.default_rng(0x5EED)
        batches = [random_batch(pkg, total, args.ranges, rng) for _ in range(args.warmup + args.steps)]
        size = max(int(b["out_off"][-1] + b["length"][-1]) for b in batches) + 16
        out_f, out_m = np.empty(size, dtype=np.uint8), np.empty(size, dtype=np.uint8)
        with pkg.SeekableArchive.from_source(ctx, path) as af, pkg.SeekableArchive(ctx, arch) as am:
            rf, rm = af.read_ranges(batches[0], out_f), am.read_ranges(batches[0], out_m)
            assert (rf["status"] == 0).all() and np.array_equal(rf, rm) and np.array_equal(out_f, out_m)
            for off, ln, oo in batches[0][:256]:
                assert np.array_equal(out_f[oo:oo + ln], plain[off:off + ln]), "a range differs from the input"
            rt = {"file": [], "memory": []}
            for i, b in enumerate(batches):
                tf = clock(lambda: af.read_ranges(b, out_f))
                tm = clock(lambda: am.read_ranges(b, out_m))
                if i >= args.warmup:
                    rt["file"].append(tf)
                    rt["memory"].append(tm)
        req = float(np.mean([int(b["length"].sum()) for b in batches[args.warmup:]]))
        line["read"] = {k: dict(stats(v), requested_GBps=req / float(np.median(v)) / GB) for k, v in rt.items()}
        line["read"].update({"ranges_per_batch": args.ranges, "range_bytes": [4096, 65536], "requested_bytes": req})
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line["value"] = line["write"]["stream"]["GBps"]
    line["unit"] = "GB/s of input, stream writer host to host"
    del fc
    ctx.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
