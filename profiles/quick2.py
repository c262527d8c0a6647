#!/usr/bin/env python3
"""Round-2 working script: per-kernel times (sequential launches, CUDA events between kernels) and whole-pass time of
the shipped launch order, per execution mode (B200Z_EXEC_MODE = warp | cta | auto), with a bit-exact check.
usage: quick2.py [config ...] ; configs: c2b c2b_small c2a1 c2a64 c3 c4 c5"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import _pkg
import datagen as G

pkg = _pkg.load()
ctx = pkg.Context(0)
if os.environ.get("B200Z_QUICK_CHECKSUM"):
    ctx.set_flags(pkg.binding.FLAG_CHECKSUM)   # so that k_xxh64 runs too
stream = torch.cuda.ExternalStream(ctx.stream())
sets = {
    "c2b": lambda: G.config_c2b(cache=False),
    "c2b_small": lambda: G.config_c2b(total_bytes=128 << 20, cache=False),
    "c2a1": lambda: G.config_c2a(total_bytes=64 << 20, nframes=1, cache=False),
    "c2a64": lambda: G.config_c2a(total_bytes=1 << 30, nframes=64, cache=False),
    "c3": lambda: G.config_c3(nframes=10000, cache=False),
    "c4": lambda: G.config_c4(nframes=1024, cache=False),
    "c4_512": lambda: G.config_c4(nframes=512, cache=False),
    "c4_2k": lambda: G.config_c4(nframes=2048, cache=False),
    "c4_4k": lambda: G.config_c4(nframes=4096, cache=False),
    "c5": lambda: G.config_c5(nframes=20000, cache=False),
}
modes = os.environ.get("QUICK_MODES", "warp,cta").split(",")
out = {}
for name in (sys.argv[1:] or ["c2b"]):
    t0 = time.time()
    fs = sets[name]()
    gen_s = time.time() - t0
    D = pkg.Dictionary.raw_content(ctx, 1, fs.raw_dict.tobytes()) if fs.raw_dict is not None else None
    for mode in modes:
        os.environ["B200Z_EXEC_MODE"] = mode
        b = pkg.Batch(ctx, fs.comp, fs.frames_io(), forced_dict=D)
        d_out = torch.zeros(fs.D + 64, dtype=torch.uint8, device="cuda")
        for _ in range(2):
            b.run(d_out)
        stream.synchronize()
        res = b.finish()
        got = d_out[:fs.D].cpu().numpy()
        ok = bool((res["status"] == 0).all()) and bool(np.array_equal(got, fs.plain))
        if not ok:
            bad = np.nonzero(res["status"] != 0)[0]
            diff = np.nonzero(got != fs.plain)[0]
            print(name, mode, "MISMATCH: failing frames", bad[:5], res[bad[:3]] if len(bad) else "", "first diff byte", diff[:5], "ndiff", len(diff), flush=True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 10
        e0.record(stream)
        for _ in range(n):
            b.run(d_out)
        e1.record(stream)
        stream.synchronize()
        ms = e0.elapsed_time(e1) / n
        profs = [b.run_profile(d_out) for _ in range(3)]
        prof = {k: float(np.median([p[k] for p in profs])) for k in profs[0]}
        tl = b.run_timeline(d_out)
        info = b.info()
        r = {"bit_exact": ok, "frames": fs.nframes, "blocks": info["blocks"], "C": fs.C, "D": fs.D, "ms": ms, "decompressed_GBps": fs.D / ms / 1e6,
             "frac_of_3350": (fs.C + fs.D) / ms / 1e6 / 3350.0, "kernel_ms": prof, "timeline_ms": tl, "sched": b.debug_sched(), "gen_s": gen_s}
        out[name + ":" + mode] = r
        print(name, mode, json.dumps(r), flush=True)
        b.close()
        del d_out
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
tag = os.environ.get("QUICK_TAG", "quick2")
json.dump(out, open(os.path.join(ROOT, "gpurun_out", tag + ".json"), "w"), indent=1)
