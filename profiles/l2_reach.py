#!/usr/bin/env python3
"""How far back k_exec's match sources reach, and what share of them an L2 can hold (CPU only, no GPU needed).

Traces a sample of frames built like C2b's (enwik-shaped text, 128 KiB single-block frames, level 3) through the oracle and
prints:
  * the distribution of match offsets (share of matches and of match bytes whose source lies within X bytes);
  * for each frames-in-flight value, the predicted share of matches whose source is still in L2 when only plaintext
    occupies it (every frame keeps the last L2 / frames bytes of its output);
  * the same under a one-priority LRU estimate, where every byte that enters L2 during the pass (plaintext, sequence records
    written and read, literals, compressed input, and the sector fills of the sources that miss) shares it: a line lives
    L2 / inflow of the pass, so a frame keeps L2 x D / (frames x inflow) bytes of its output, solved as a fixed point;
  * the DRAM bytes of the source misses that follow, per pass of the full workload.
A model, not a measurement: it ignores L1 hits, the split of the H100's L2 into two partitions, and frames that start and
finish at different times.

    python profiles/l2_reach.py [--frames 16] [--l2-mib 50] [--sms 132]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FRAME = 131072
C2B_FRAMES = 8192
WARPS_PER_CTA = 4   # k_exec: one frame per warp


def trace_frames(n):
    import datagen as G
    from oracle import oracle as O
    fs = G.config_c2b(total_bytes=n * FRAME, frame_bytes=FRAME, cache=False)
    offs, mls, srcs, recs, lits = [], [], [], 0, 0
    for i in range(fs.nframes):
        frame = fs.comp[int(fs.src_off[i]):int(fs.src_off[i] + fs.src_size[i])].tobytes()
        d = O.FrameDecoder()
        d.trace_enable()
        r = d.reset(frame)
        d.decode_blocks(r)
        blocks, _lits, seqs = d.trace()
        for b in blocks:
            if b["block_type"] != 2:
                continue
            s = seqs[b["seq_offset"]:b["seq_offset"] + b["num_sequences"]].astype(np.int64)
            pos = b["out_offset"] + np.cumsum(s[:, 0] + s[:, 1]) - s[:, 1]   # frame position where each match starts
            m = s[:, 1] > 0
            offs.append(s[m, 3]); mls.append(s[m, 1]); srcs.append(pos[m] - s[m, 3])
            recs += 12 * len(s)
            lits += b["regenerated_size"]
    return fs, np.concatenate(offs), np.concatenate(mls), np.concatenate(srcs), recs, lits


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--l2-mib", type=float, default=50.0)
    ap.add_argument("--sms", type=int, default=132)
    args = ap.parse_args()
    fs, off, ml, src, rec_b, lit_b = trace_frames(args.frames)
    D = fs.D
    sectors = ((src & 31) + ml + 31) // 32 * 32   # bytes a missing source brings in, whole 32-byte sectors
    scale = C2B_FRAMES * FRAME / D
    print(f"{fs.nframes} frames, {len(off)} matches, {D / len(off):.1f} output bytes per match, mean match length {ml.mean():.1f}")
    print(f"match offset: median {np.median(off) / 1024:.1f} KiB, quartiles {np.percentile(off, 25) / 1024:.1f} / {np.percentile(off, 75) / 1024:.1f} KiB, "
          f"90th percentile {np.percentile(off, 90) / 1024:.1f} KiB\n")
    cut = [2, 4, 8, 16, 24, 32, 64]
    print("| match source within | " + " | ".join(f"{k} KiB" for k in cut) + " |")
    print("|---|" + "---|" * len(cut))
    print("| share of matches | " + " | ".join(f"{100 * np.mean(off <= k * 1024):.1f} %" for k in cut) + " |")
    print("| share of match bytes | " + " | ".join(f"{100 * ml[off <= k * 1024].sum() / ml.sum():.1f} %" for k in cut) + " |\n")

    L2 = args.l2_mib * 2**20
    Dt = C2B_FRAMES * FRAME
    streams = scale * (2 * rec_b + lit_b + float(fs.C))   # records written + read, literals, compressed input (full workload)
    print(f"L2 {args.l2_mib:.0f} MiB; per pass of {C2B_FRAMES} frames: plaintext {Dt / 1e9:.2f} GB, streamed {streams / 1e9:.2f} GB "
          f"(records {2 * scale * rec_b / 1e9:.2f} written + read, literals {scale * lit_b / 1e9:.2f}, input {scale * fs.C / 1e9:.2f})\n")
    print("| CTAs per SM | frames in flight | plaintext only: reach, source hits | one priority (LRU): reach, source hits | source-miss DRAM GB per pass, plaintext only / one priority |")
    print("|---|---|---|---|---|")
    for c in (6, 5, 4, 3):
        F = args.sms * c * WARPS_PER_CTA
        r_p = L2 / F
        miss_p = scale * sectors[off > r_p].sum()
        r = r_p
        for _ in range(100):   # fixed point: the misses' fills are inflow too
            miss = scale * sectors[off > r].sum()
            r = 0.5 * r + 0.5 * L2 * Dt / (F * (Dt + streams + miss))
        miss = scale * sectors[off > r].sum()
        print(f"| {c} | {F} | {r_p / 1024:.1f} KiB, {100 * np.mean(off <= r_p):.1f} % | {r / 1024:.1f} KiB, {100 * np.mean(off <= r):.1f} % | "
              f"{miss_p / 1e9:.2f} / {miss / 1e9:.2f} |")


if __name__ == "__main__":
    main()
