#!/usr/bin/env python3
"""bench_decode_all.py -- decode_all on the batch path (b200z_decode_all_prepare + b200z_batch_run): a buffer of concatenated frames
decoded in one GPU submission, without the caller's frame offsets.

    python bench_decode_all.py [--steps K] [--warmup W] [--configs c2b,c4,c5] [--tier2-frames N]

For each workload (C2b: 8,192 frames of 128 KiB; C4: 4,096 frames of 1 MiB; C5: 100,000 small frames with their raw-content dictionary
forced), `comp` is one device buffer.  Reports, per workload:
  - prepare: wall milliseconds of b200z_decode_all_prepare on device input, and the device milliseconds of k_find_frames and of the
    candidate walk (k_walk, count pass), from torch.profiler;
  - decode_all: b200z_batch_run milliseconds (CUDA events, median of the steps) and GB/s of plaintext, alternated step by step in
    the same process with the known-offset Batch on the same frames (bench.py's `value` path);
  - tier2: the FrameDecoder.decode_all mirror on the host buffer of the first --tier2-frames frames.
Every output must equal `plain`.  Prints one JSON line with the card's name and power limit.  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_compress import card_info  # noqa: E402

GB = 1e9


def kernel_ms(prof, name):
    return sum(e.device_time_total for e in prof.key_averages() if name in e.key) / 1e3


def run_config(pkg, name, fs, args):
    import torch
    ctx = pkg.Context(0)
    D = pkg.Dictionary.raw_content(ctx, 1, fs.raw_dict.tobytes()) if fs.raw_dict is not None else None
    d_in = torch.from_numpy(fs.comp).cuda()
    total = int(fs.D)
    out = torch.zeros(total + 16, dtype=torch.uint8, device="cuda")
    plain = torch.from_numpy(fs.plain).cuda()
    torch.cuda.synchronize()
    # prepare (device input): wall time, then once more under the profiler for the discovery kernels
    t0 = time.perf_counter()
    ab = pkg.AllBatch(ctx, d_in, forced_dict=D)
    prep_ms = (time.perf_counter() - t0) * 1e3
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA], acc_events=True) as prof:
        pkg.AllBatch(ctx, d_in, forced_dict=D).close()
        torch.cuda.synchronize()
    find_ms, walk_ms = kernel_ms(prof, "k_find_frames"), kernel_ms(prof, "k_walk")
    io = np.zeros(fs.nframes, dtype=pkg.binding.FRAME_IO_DTYPE)
    io["src_off"], io["src_size"], io["out_off"], io["out_cap"] = fs.src_off, fs.src_size, fs.out_off, fs.out_size
    kb = pkg.Batch(ctx, d_in, io, forced_dict=D)
    stream = torch.cuda.ExternalStream(ctx.stream())

    def once(b):
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        b.run(out[:total])
        z.record(stream)
        z.synchronize()
        return a.elapsed_time(z)

    for _ in range(args.warmup):
        once(ab); once(kb)
    t_all, t_known = [], []
    for _ in range(args.steps):
        t_all.append(once(ab))
        t_known.append(once(kb))
    once(ab)
    s, _res = ab.finish()
    assert s["status"] == 0 and s["written"] == total and torch.equal(out[:total], plain), f"{name}: decode_all output differs from plain"
    once(kb)
    assert (kb.finish()["status"] == 0).all() and torch.equal(out[:total], plain)
    m_all, m_known = float(np.median(t_all)), float(np.median(t_known))
    line = {"frames": fs.nframes, "compressed_bytes": int(fs.comp.size), "plain_bytes": total, "prepare_ms": prep_ms,
            "k_find_frames_ms": find_ms, "candidate_walk_ms": walk_ms, "candidates_launches": ab.info()["launches_per_run"],
            "decode_all_ms": m_all, "decode_all_GBps": total / (m_all / 1e3) / GB,
            "decode_all_ms_min_max": [min(t_all), max(t_all)], "known_offsets_ms": m_known, "known_offsets_GBps": total / (m_known / 1e3) / GB,
            "known_offsets_ms_min_max": [min(t_known), max(t_known)], "ratio_decode_all_over_known": m_all / m_known}
    ab.close(); kb.close()
    # tier 2: the FrameDecoder mirror's decode_all (host loop, one block per submission) on a subset
    n2 = min(args.tier2_frames, fs.nframes)
    if n2 and D is None:
        end = int(fs.src_off[n2 - 1] + fs.src_size[n2 - 1])
        sub = fs.comp[:end].tobytes()
        want = int(fs.out_off[n2 - 1] + fs.out_size[n2 - 1])
        dec = pkg.FrameDecoder(ctx)
        t0 = time.perf_counter()
        got = dec.decode_all(sub, want)
        dt = time.perf_counter() - t0
        assert got == fs.plain[:want].tobytes(), f"{name}: tier-2 decode_all differs from plain"
        line["tier2"] = {"frames": n2, "plain_bytes": want, "ms": dt * 1e3, "GBps": want / dt / GB}
    ctx.close()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--configs", default="c2b,c4,c5")
    ap.add_argument("--tier2-frames", type=int, default=256)
    ap.add_argument("--c4-frames", type=int, default=4096)
    args = ap.parse_args()
    import torch
    import _pkg
    import datagen as G
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode_all.py needs a CUDA device: the product path has no CPU fallback")
    pkg = _pkg.load()
    makers = {"c2b": lambda: G.config_c2b(), "c4": lambda: G.config_c4(nframes=args.c4_frames), "c5": lambda: G.config_c5()}
    line = {"metric": "decode_all_GBps", "unit": "GB/s", "card": card_info(), "steps": args.steps}
    for name in args.configs.split(","):
        line[name] = run_config(pkg, name, makers[name](), args)
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())
