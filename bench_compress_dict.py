#!/usr/bin/env python3
"""bench_compress_dict.py -- input GB/s of the batch compressor against a dictionary (b200z_compress_frames_batch_dict, ruzstd's
Fastest level, checksum on).

    python bench_compress_dict.py [--steps K] [--warmup W] [--nframes N] [--frames-per-call F] [--skip-cpu] [--finalize]

The workload is C5 (datagen.config_c5: 100,000 frames of 1-8 KiB drawn mostly from a 112,640-byte raw-content dictionary),
device-resident, in submissions of at most 20,000 frames (--frames-per-call).  Before timing, the frames are decoded on the GPU
with the dictionary forced and must equal the input.  Prints one JSON line: input GB/s (CUDA events around the submissions,
median of the steps), the ratio, each kernel's milliseconds and k_cdict's
(the dictionary's match table, built once), the same frames without the dictionary, the card's name and power limit, and
`cpu_baseline`: libzstd level 1 and 3 with the dictionary as a CDict built once, one thread and all host threads.  Nothing is
written to the tree.

--finalize adds a "finalize" record: b200z_dict_finalize of the C5 content on samples 0-97,999 (device time of the call, CUDA
events on the context's stream; median of --steps calls), then the held-out last 2,000 frames and all of C5 compressed with the
finalized dictionary, with and without its entropy tables (dict_tables; ratio, GB/s), beside libzstd levels 1 and 3 with ZDICT_finalizeDictionary's dictionary of the same content
on the same samples (ratio on the held-out frames).
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

GB = 1e9


def libzstd_cdict_baseline(pieces, content, level):
    """libzstd with `content` as a CDict at `level` (one frame per piece, checksum on as in the GPU runs): one thread on the first
    2,000 pieces, and all host threads on all of them."""
    import datagen
    from concurrent.futures import ThreadPoolExecutor
    z = datagen.zstd()
    z.ZSTD_createCDict.restype = C.c_void_p; z.ZSTD_createCDict.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    z.ZSTD_freeCDict.argtypes = [C.c_void_p]
    z.ZSTD_CCtx_refCDict.restype = C.c_size_t; z.ZSTD_CCtx_refCDict.argtypes = [C.c_void_p, C.c_void_p]
    cdict = z.ZSTD_createCDict(content, len(content), level)

    def run(chunk):
        cctx = z.ZSTD_createCCtx()
        z.ZSTD_CCtx_refCDict(cctx, cdict)
        z.ZSTD_CCtx_setParameter(cctx, datagen.ZSTD_c_checksumFlag, 1)
        dst = np.empty(z.ZSTD_compressBound(8192 * 2), dtype=np.uint8)
        out = 0
        for p in chunk:
            n = z.ZSTD_compress2(cctx, dst.ctypes.data, dst.nbytes, p, len(p))
            assert not z.ZSTD_isError(n)
            out += n
        z.ZSTD_freeCCtx(cctx)
        return out
    sub = pieces[:2000]
    t0 = time.perf_counter()
    n1 = run(sub)
    one = sum(len(p) for p in sub) / (time.perf_counter() - t0) / GB
    threads = bench.host_threads()
    chunks = [pieces[i::threads] for i in range(threads)]
    with ThreadPoolExecutor(max_workers=threads) as ex:
        t0 = time.perf_counter()
        sizes = list(ex.map(run, chunks))
        dt = time.perf_counter() - t0
    z.ZSTD_freeCDict(cdict)
    total = sum(len(p) for p in pieces)
    return {"kind": f"libzstd level {level}, CDict", "one_core_GBps": one, "one_core_ratio": sum(len(p) for p in sub) / n1,
            "all_cores_GBps": total / dt / GB, "cores": threads, "ratio": total / sum(sizes)}


def cdict_ms(pkg, ctx, content, d_in, io, d_out):
    """k_cdict's device time, from torch.profiler around the first compression with a fresh dictionary."""
    import torch
    D = pkg.Dictionary.raw_content(ctx, 1, content)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        pkg.compress_frames(ctx, d_in, io[:1], d_out, dict=D)
        torch.cuda.synchronize()
    ms = [e.device_time_total / 1e3 for e in prof.key_averages() if "k_cdict" in e.key]
    return ms[0] if ms else None


def compress_all(pkg, ctx, d_in, subs, d_out, dict, prof=None, tables=False):
    """Every submission in turn; the results of all frames.  With `prof`, adds each kernel's milliseconds to it."""
    res = []
    for io in subs:
        res.append(pkg.compress_frames(ctx, d_in, io, d_out, dict=dict, dict_tables=tables))
        if prof is not None:
            for k, v in pkg.compress_profile(ctx).items():
                prof[k] = prof.get(k, 0.0) + v
    return np.concatenate(res)


def timed(pkg, ctx, d_in, subs, d_out, dict, steps, warmup, tables=False):
    import torch
    for _ in range(warmup):
        compress_all(pkg, ctx, d_in, subs, d_out, dict, tables=tables)
    stream = torch.cuda.ExternalStream(ctx.stream())
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        res = compress_all(pkg, ctx, d_in, subs, d_out, dict, tables=tables)
        b.record(stream)
        b.synchronize()
        times.append(a.elapsed_time(b) / 1e3)
    ctx.set_flags(pkg.binding.FLAG_PROFILE)
    prof = {}
    compress_all(pkg, ctx, d_in, subs, d_out, dict, prof, tables)
    ctx.set_flags(0)
    return float(np.median(times)), times, prof, res


def zdict_finalize(content, pieces, level=3):
    """ZDICT_finalizeDictionary(content, samples = pieces), with the ID libzstd derives from the content."""
    import datagen
    z = datagen.zstd()

    class Params(C.Structure):
        _fields_ = [("compressionLevel", C.c_int), ("notificationLevel", C.c_uint), ("dictID", C.c_uint)]
    z.ZDICT_finalizeDictionary.restype = C.c_size_t
    z.ZDICT_finalizeDictionary.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint, Params]
    z.ZDICT_isError.restype = C.c_uint
    z.ZDICT_isError.argtypes = [C.c_size_t]
    buf = np.frombuffer(b"".join(pieces), dtype=np.uint8)
    sizes = np.array([len(p) for p in pieces], dtype=np.uintp)
    out = np.zeros(len(content) + 4096, dtype=np.uint8)
    n = z.ZDICT_finalizeDictionary(out.ctypes.data, out.size, content, len(content), buf.ctypes.data, sizes.ctypes.data, len(pieces),
                                   Params(level, 0, 0))
    assert not z.ZDICT_isError(n)
    return out[:n].tobytes()


def finalize_arm(pkg, ctx, fs, content, d_in, io, subs, d_out, steps, warmup):
    """b200z_dict_finalize on samples 0-97,999 (at most all but the last 2,000), and the finalized dictionary in use."""
    import torch
    import datagen
    n = fs.nframes
    ntrain = max(0, min(98000, n - 2000))
    plain = fs.plain
    pieces = [plain[int(o):int(o + k)].tobytes() for o, k in zip(fs.out_off, fs.out_size)]
    t0 = int(fs.out_off[0]) if n else 0
    t1 = int(fs.out_off[ntrain - 1] + fs.out_size[ntrain - 1]) if ntrain else t0
    train = d_in[t0:t1]
    sizes = fs.out_size[:ntrain].astype(np.uint64)
    stream = torch.cuda.ExternalStream(ctx.stream())
    for _ in range(warmup):
        d = pkg.finalize_dict(ctx, content, train, sizes)
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        d = pkg.finalize_dict(ctx, content, train, sizes)
        b.record(stream)
        b.synchronize()
        times.append(a.elapsed_time(b))
    D = pkg.Dictionary.decode_dict(ctx, d)
    caps = np.array([pkg.compress_bound(int(k), D) for k in fs.out_size], dtype=np.uint64)
    assert (caps <= io["dst_cap"] + 4).all()
    io2 = io.copy()
    io2["dst_cap"] = caps
    io2["dst_off"] = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.uint64)
    out2 = torch.empty(int(caps.sum()), dtype=torch.uint8, device="cuda")
    held = io2[ntrain:]
    subs2 = [io2[i:i + len(subs[0])] for i in range(0, len(io2), len(subs[0]))]
    held_in, all_in = int(fs.out_size[ntrain:].sum()), int(fs.out_size.sum())
    arms = {}
    for name, tables in (("without_tables", False), ("dict_tables", True)):
        th, _, _, rh = timed(pkg, ctx, d_in, [held], out2, D, steps, warmup, tables)
        ta, _, _, ra = timed(pkg, ctx, d_in, subs2, out2, D, steps, warmup, tables)
        arms[name] = {"held_out": {"frames": n - ntrain, "ratio": held_in / int(rh["dst_size"].sum()), "GBps": held_in / th / GB},
                      "all": {"ratio": all_in / int(ra["dst_size"].sum()), "GBps": all_in / ta / GB}}
    zd = zdict_finalize(content, pieces[:ntrain])
    z = {f"libzstd_level{lv}_held_out_ratio": held_in / sum(len(datagen.compress(p, level=lv, raw_dict=zd)) for p in pieces[ntrain:])
         for lv in (1, 3)}
    return {"samples": ntrain, "dict_bytes": len(d), "header_bytes": len(d) - len(content), "ms": float(np.median(times)),
            "ms_min_max": [min(times), max(times)], **arms, "zdict_header_bytes": len(zd) - len(content), **z}


def run(args):
    import torch
    import _pkg
    import datagen
    if not torch.cuda.is_available():
        raise SystemExit("bench_compress_dict.py needs a CUDA device: the product path has no CPU fallback")
    pkg = _pkg.load()
    ctx = pkg.Context(0)
    fs = datagen.config_c5(nframes=args.nframes)
    content = fs.raw_dict.tobytes()
    plain = fs.plain
    total = int(plain.size)
    D = pkg.Dictionary.raw_content(ctx, 1, content)
    io = np.zeros(fs.nframes, dtype=pkg.binding.COMPRESS_IO_DTYPE)
    caps = np.array([pkg.compress_bound(int(n), D) for n in fs.out_size], dtype=np.uint64)
    io["src_off"], io["src_size"], io["dst_cap"] = fs.out_off, fs.out_size, caps
    io["dst_off"] = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.uint64)
    d_in = torch.from_numpy(plain).cuda()
    d_out = torch.empty(int(caps.sum()), dtype=torch.uint8, device="cuda")
    # the compressor stages 128 KiB of literals and room for 26,224 sequences per block whatever the block's size, so 100,000
    # small frames go in submissions of at most --frames-per-call frames
    subs = [io[i:i + args.frames_per_call] for i in range(0, len(io), args.frames_per_call)]
    res = compress_all(pkg, ctx, d_in, subs, d_out, D)
    assert (res["status"] == 0).all()
    dio = np.zeros(fs.nframes, dtype=pkg.binding.FRAME_IO_DTYPE)
    dio["src_off"], dio["src_size"], dio["out_off"], dio["out_cap"] = io["dst_off"], res["dst_size"], io["src_off"], io["src_size"]
    back = torch.empty(total + 16, dtype=torch.uint8, device="cuda")
    dres = pkg.decode_frames(ctx, d_out, dio, back, forced_dict=D)
    assert (dres["status"] == 0).all() and torch.equal(back[:total], d_in), "GPU decode of the compressed frames differs from the input"
    del back
    line = {"metric": "compress_dict_GBps", "unit": "GB/s", "level": "Fastest", "checksum": True, "card": card_info(), "config": "C5",
            "frames": fs.nframes, "frames_per_call": args.frames_per_call, "input_bytes": total, "dict_bytes": len(content)}
    t, times, prof, res = timed(pkg, ctx, d_in, subs, d_out, D, args.steps, args.warmup)
    out_bytes = int(res["dst_size"].sum())
    line.update({"value": total / t / GB, "ms": t * 1e3, "ms_min_max": [min(times) * 1e3, max(times) * 1e3], "ratio": total / out_bytes,
                 "output_bytes": out_bytes, "kernel_ms": prof, "k_cdict_ms": cdict_ms(pkg, ctx, content, d_in, io, d_out),
                 "raw_blocks": int(res["raw_blocks"].sum()), "rle_blocks": int(res["rle_blocks"].sum())})
    t0, times0, prof0, res0 = timed(pkg, ctx, d_in, subs, d_out, None, args.steps, args.warmup)
    line["no_dict"] = {"value": total / t0 / GB, "ms": t0 * 1e3, "ratio": total / int(res0["dst_size"].sum()), "kernel_ms": prof0}
    if args.finalize:
        line["finalize"] = finalize_arm(pkg, ctx, fs, content, d_in, io, subs, d_out, args.steps, args.warmup)
    if not args.skip_cpu:
        pieces = [plain[int(o):int(o + n)].tobytes() for o, n in zip(fs.out_off, fs.out_size)]
        line["cpu_baseline"] = [libzstd_cdict_baseline(pieces, content, lv) for lv in (1, 3)]
    ctx.close()
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--nframes", type=int, default=100000)
    ap.add_argument("--frames-per-call", type=int, default=20000)
    ap.add_argument("--skip-cpu", action="store_true")
    ap.add_argument("--finalize", action="store_true", help="add the b200z_dict_finalize arm")
    run(ap.parse_args())
    return 0


if __name__ == "__main__":
    sys.exit(main())
