#!/usr/bin/env python3
"""bench_dict_train.py -- the raw-content dictionary trainer (b200z_dict_train_raw) on all of C5.

    python bench_dict_train.py [--steps K] [--warmup W] [--nframes N] [--segment-sizes 2048,256] [--skip-cpu]

Trains on the C5 plaintext (datagen.config_c5: 100,000 samples of 1-8 KiB, device-resident) into a 112,640-byte dictionary at
each segment size L of --segment-sizes (default 2048 and 256).  Prints one JSON line with, per L: device ms (CUDA events around the call, median of the steps),
input GB/s, kernel launches per call, each kernel's device ms (torch.profiler, a separate run), libzstd's
ZDICT_trainFromBuffer_fastCover on the same input (d = 8, k = L; nbThreads 1 and all usable cores), and the held-out ratio:
dictionaries trained on all samples but the last 2,000, applied to those 2,000 by libzstd level 3 (raw dictionary) and by this
library's compressor (dict=).  The card's name and power limit are read in the same call.  Nothing is written to the tree.
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

import bench  # noqa: E402  (host_threads)
from bench_compress import card_info  # noqa: E402

DICT = 112640
HELD = 2000


class ZParams(C.Structure):
    _fields_ = [("compressionLevel", C.c_int), ("notificationLevel", C.c_uint), ("dictID", C.c_uint)]


class FastCoverParams(C.Structure):
    _fields_ = [("k", C.c_uint), ("d", C.c_uint), ("f", C.c_uint), ("steps", C.c_uint), ("nbThreads", C.c_uint), ("splitPoint", C.c_double),
                ("accel", C.c_uint), ("shrinkDict", C.c_uint), ("shrinkDictMaxRegression", C.c_uint), ("zParams", ZParams)]


def fastcover(plain, sizes, L, threads):
    """(seconds, content-only dictionary) of ZDICT_trainFromBuffer_fastCover with d = 8, k = L, f = 20, accel = 1."""
    import datagen
    z = datagen.zstd()
    fn = z.ZDICT_trainFromBuffer_fastCover
    fn.restype = C.c_size_t
    fn.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint, FastCoverParams]
    z.ZDICT_isError.restype = C.c_uint
    z.ZDICT_isError.argtypes = [C.c_size_t]
    z.ZDICT_getDictHeaderSize.restype = C.c_size_t
    z.ZDICT_getDictHeaderSize.argtypes = [C.c_void_p, C.c_size_t]
    sz = np.ascontiguousarray(sizes, dtype=np.uintp)
    out = np.zeros(DICT, dtype=np.uint8)
    p = FastCoverParams(k=L, d=8, f=20, steps=0, nbThreads=threads, splitPoint=1.0, accel=1, shrinkDict=0, shrinkDictMaxRegression=0,
                        zParams=ZParams(3, 0, 0))
    t0 = time.perf_counter()
    n = fn(out.ctypes.data, DICT, plain.ctypes.data, sz.ctypes.data, len(sz), p)
    dt = time.perf_counter() - t0
    assert not z.ZDICT_isError(n)
    h = z.ZDICT_getDictHeaderSize(out.ctypes.data, n)
    return dt, out[h:n].tobytes()


def ratio_libzstd(pieces, content):
    import datagen
    return sum(len(p) for p in pieces) / sum(len(datagen.compress(p, level=3, raw_dict=content)) for p in pieces)


def ratio_own(pkg, ctx, pieces, content):
    D = pkg.Dictionary.raw_content(ctx, 1, content) if content is not None else None
    io = np.zeros(len(pieces), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    so = oo = 0
    for i, p in enumerate(pieces):
        cap = pkg.compress_bound(len(p), D)
        io[i] = (so, len(p), oo, cap)
        so += len(p)
        oo += cap
    out = np.zeros(oo, dtype=np.uint8)
    res = pkg.compress_frames(ctx, np.frombuffer(b"".join(pieces), dtype=np.uint8), io, out, checksum=False, dict=D)
    assert (res["status"] == 0).all()
    return so / int(res["dst_size"].sum())


def kernel_ms(pkg, ctx, d_plain, sizes, L):
    import torch
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        pkg.create_raw_dict(ctx, d_plain, DICT, sizes, segment_size=L)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ("k_dtcount", "k_dtprev", "k_dtepoch"):
            if k in e.key:
                out[k] = out.get(k, 0.0) + e.device_time_total / 1e3
    return out


def run(args):
    import torch
    import _pkg
    import datagen
    if not torch.cuda.is_available():
        raise SystemExit("bench_dict_train.py needs a CUDA device: the product path has no CPU fallback")
    pkg = _pkg.load()
    ctx = pkg.Context(0)
    fs = datagen.config_c5(nframes=args.nframes)
    plain = fs.plain
    sizes = fs.out_size.astype(np.uint64)
    total = int(plain.size)
    d_plain = torch.from_numpy(plain).cuda()
    stream = torch.cuda.ExternalStream(ctx.stream())
    line = {"metric": "dict_train_ms", "unit": "ms", "card": card_info(), "config": "C5", "samples": int(len(sizes)), "input_bytes": total,
            "dict_bytes": DICT, "runs": {}}
    pieces = [plain[int(o):int(o + n)].tobytes() for o, n in zip(fs.out_off, fs.out_size)]
    held = pieces[-HELD:]
    cut = int(fs.out_off[-HELD])
    no_dict = {"libzstd_l3": ratio_libzstd(held, None), "own": ratio_own(pkg, ctx, held, None)}
    for L in [int(x) for x in args.segment_sizes.split(",")]:
        host = pkg.create_raw_dict(ctx, plain, DICT, sizes, segment_size=L, segments=True)
        dev = pkg.create_raw_dict(ctx, d_plain, DICT, sizes, segment_size=L, segments=True)
        assert host[0] == dev[0] and (host[1] == dev[1]).all(), "host and device input give different dictionaries"
        for _ in range(args.warmup):
            pkg.create_raw_dict(ctx, d_plain, DICT, sizes, segment_size=L)
        times = []
        for _ in range(args.steps):
            before = ctx.kernel_launches()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            pkg.create_raw_dict(ctx, d_plain, DICT, sizes, segment_size=L)
            b.record(stream)
            b.synchronize()
            times.append(a.elapsed_time(b))
            launches = ctx.kernel_launches() - before
        ms = float(np.median(times))
        r = {"ms": ms, "ms_min_max": [min(times), max(times)], "input_GBps": total / ms / 1e6, "launches": int(launches),
             "epochs": int(len(dev[1])), "kernel_ms": kernel_ms(pkg, ctx, d_plain, sizes, L)}
        train_d = pkg.create_raw_dict(ctx, d_plain[:cut], DICT, sizes[:-HELD], segment_size=L)
        r["heldout"] = {"libzstd_l3": ratio_libzstd(held, train_d), "own": ratio_own(pkg, ctx, held, train_d)}
        if not args.skip_cpu:
            cores = bench.host_threads()
            t1, _ = fastcover(plain, sizes, L, 1)
            tn, _ = fastcover(plain, sizes, L, cores)
            _, fc = fastcover(plain[:cut], sizes[:-HELD], L, cores)
            r["fastcover"] = {"s_one_thread": t1, "s_all_cores": tn, "cores": cores, "heldout_libzstd_l3": ratio_libzstd(held, fc)}
        line["runs"][str(L)] = r
    line["heldout_no_dict"] = no_dict
    line["heldout_generator_dict_libzstd_l3"] = ratio_libzstd(held, fs.raw_dict.tobytes())
    ctx.close()
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--nframes", type=int, default=100000)
    ap.add_argument("--segment-sizes", default="2048,256")
    ap.add_argument("--skip-cpu", action="store_true")
    run(ap.parse_args())
    return 0


if __name__ == "__main__":
    sys.exit(main())
