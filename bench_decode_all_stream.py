#!/usr/bin/env python3
"""bench_decode_all_stream.py -- plaintext GB/s of decode_all from a reader to a writer (b200z_decode_all_stream, tier 1d), host
memory to host memory, against the batch path, the tier-2 mirror and the host work alone.

    python bench_decode_all_stream.py [--steps K] [--workloads a,b,c]

Workloads:
  a  C2b: 8192 frames of 128 KiB of enwik9-shaped text back to back (datagen.config_c2b)
  b  one frame of the same 1 GiB of text written by FrameCompressor (no Frame_Content_Size, 8192 chained blocks): the block chain
     of one frame, carried from submission to submission
  c  C5: small frames against a raw-content dictionary (datagen.config_c5), with forced_dict
Arms, alternated step by step in one run, wall time around each call:
  stream     decode_all_stream at the default chunk; its read and write callbacks memmove from the compressed bytes and into a
             preallocated host buffer
  batch      decode_frames host to host with the frames' offsets known (the pipelined batch path: the upper bound)
  tier2      FrameDecoder.decode_all on the first 256 frames (a, c), StreamingDecoder.read_to_end on a 32 MiB frame of the text (b)
  host_only  the stream arm's read and write callbacks over the same bytes, with no decode
Prints one JSON line: per workload and arm the median and min-max GB/s of plaintext, kernel launches and submissions per call, the
stream's ratio to batch and to host_only, the device memory decode_all_stream holds (free device memory before and after its first
call), and the card's name and power limit.  Outputs are checked against the plaintext outside the timed region.  Nothing is
written to the tree.
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

GB = 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--workloads", default="a,b,c")
    args = ap.parse_args()
    import torch
    import _pkg
    import datagen
    from bench_compress import card_info
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode_all_stream.py needs a CUDA device: the product path has no CPU fallback")
    pkg = _pkg.load()
    B = pkg.binding
    L = pkg.lib()
    ctx = pkg.Context(0)

    def workload(name):
        if name == "a":
            fs = datagen.config_c2b()
            return fs.comp, fs.plain, fs.frames_io(), None, fs
        if name == "b":
            plain = datagen.c2_text_plain(1 << 30)
            out = bytearray()
            pkg.compress(ctx, plain.tobytes(), out)
            comp = np.frombuffer(bytes(out), dtype=np.uint8)
            io = np.array([(0, len(comp), 0, len(plain))], dtype=B.FRAME_IO_DTYPE)
            return comp, plain, io, None, None
        fs = datagen.config_c5()
        return fs.comp, fs.plain, fs.frames_io(), pkg.Dictionary.raw_content(ctx, 1, fs.raw_dict), fs

    result, held = {}, None
    for name in args.workloads.split(","):
        comp, plain, io, D, fs = workload(name)
        total = int(io["out_cap"].sum()) if fs is not None else len(plain)
        plain_v = np.asarray(plain, dtype=np.uint8)[:total]
        out = np.empty(total + 16, dtype=np.uint8)
        src_addr, n_comp = comp.ctypes.data, len(comp)
        pos = {"r": 0, "w": 0}

        def _read(_u, buf, n):
            k = min(n, n_comp - pos["r"])
            C.memmove(buf, src_addr + pos["r"], k)
            pos["r"] += k
            return k

        def _write(_u, buf, n):
            C.memmove(out.ctypes.data + pos["w"], buf, n)
            pos["w"] += n
            return n

        rd, wr = B.READ_FN(_read), B.WRITE_FN(_write)
        res = np.zeros(1, dtype=B.STREAM_RESULT_DTYPE)
        darr, nd, forced = B._dict_args([], D)

        def stream():
            pos["r"] = pos["w"] = 0
            ctx._chk(L.b200z_decode_all_stream(ctx.h, rd, None, wr, None, darr, nd, forced, 0, res.ctypes.data))
            assert res[0]["all"]["status"] == 0
            return int(res[0]["all"]["written"])

        bout = np.empty(total + 16, dtype=np.uint8)

        def batch():
            r = pkg.decode_frames(ctx, comp, io, bout, forced_dict=D)
            return int(r["out_size"].sum())

        if name == "b":
            t2_plain = plain_v[:32 << 20].tobytes()
            t2b = bytearray()
            pkg.compress(ctx, t2_plain, t2b)
            t2_comp = bytes(t2b)

            def tier2():
                got = pkg.StreamingDecoder(ctx, t2_comp).read_to_end()
                assert got == t2_plain
                return len(got)
        else:
            nt2 = min(256, len(io))
            t2_comp = comp[:int(io[nt2 - 1]["src_off"] + io[nt2 - 1]["src_size"])].tobytes()
            t2_len = int(io[:nt2]["out_cap"].sum())

            def tier2():
                d = pkg.FrameDecoder(ctx)
                if D is not None:
                    d.add_raw_content_dict(1, fs.raw_dict)
                    got = bytearray()
                    for i in range(nt2):   # forced dictionary: one frame at a time, as the reference needs force_dict after init
                        f = comp[int(io[i]["src_off"]):int(io[i]["src_off"] + io[i]["src_size"])].tobytes()
                        r = d.reset(f)
                        d.force_dict(1)
                        d.decode_blocks(r)
                        got += d.collect()
                    return len(got)
                return len(d.decode_all(t2_comp, t2_len))

        pinned = torch.empty(64 << 20, dtype=torch.uint8).pin_memory()
        pin = pinned.data_ptr()

        def host_only():
            pos["r"] = pos["w"] = 0
            while _read(None, pin, 64 << 20):
                pass
            left = total
            while left:
                n = min(64 << 20, left)
                _write(None, pin, n)
                left -= n
            return total

        if held is None:
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info(0)[0]
            stream()
            held = free0 - torch.cuda.mem_get_info(0)[0]
        # outputs against the plaintext, outside the timing
        assert stream() == total and np.array_equal(out[:total], plain_v), f"{name}: stream output differs"
        assert batch() == total and np.array_equal(bout[:total], plain_v), f"{name}: batch output differs"
        arms = {"stream": stream, "batch": batch, "tier2": tier2, "host_only": host_only}
        for f in arms.values():
            f()
        times = {k: [] for k in arms}
        sizes, launches, subs = {}, {}, None
        for _ in range(args.steps):
            for k, f in arms.items():
                l0 = ctx.kernel_launches()
                t0 = time.perf_counter()
                sizes[k] = f()
                times[k].append(time.perf_counter() - t0)
                launches[k] = ctx.kernel_launches() - l0
                if k == "stream":
                    subs = int(res[0]["submissions"])
        arms_out = {}
        for k, ts in times.items():
            t = float(np.median(ts))
            arms_out[k] = {"GBps": sizes[k] / t / GB, "GBps_min_max": [sizes[k] / max(ts) / GB, sizes[k] / min(ts) / GB], "ms": t * 1e3,
                           "plaintext_bytes": sizes[k], "kernel_launches": launches[k]}
        s = arms_out["stream"]["GBps"]
        print(name, json.dumps(arms_out), file=sys.stderr)
        result[name] = {"arms": arms_out, "stream_submissions": subs, "compressed_bytes": n_comp,
                        "stream_over_tier2": s / arms_out["tier2"]["GBps"], "stream_over_batch": s / arms_out["batch"]["GBps"],
                        "stream_over_host_only": s / arms_out["host_only"]["GBps"]}
        del comp, plain, out, bout
    line = {"metric": "decode_all_stream_GBps", "unit": "GB/s", "value": result.get("a", next(iter(result.values())))["arms"]["stream"]["GBps"],
            "steps": args.steps, "chunk_bytes": 64 << 20, "card": card_info(), "workloads": result, "stream_device_bytes_held": int(held)}
    ctx.close()
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())
