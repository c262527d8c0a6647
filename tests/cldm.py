"""Long-distance matching (window_log > 17, an extension) written out plainly: what the long-match kernels (csrc/ldm.cu) must find,
what k_cmatch<DICT, LAZY, true> must then produce for every block, and the frame the compressor must write.

This module restates the rules of DESIGN.md section 4.11 in Python, calling nothing in the library.  It keeps the Fastest and LAZY
models' blocks, hashes, tables, segments, rounds and packing (tests/cparse.py, tests/clazy.py) and adds:

  frames    only frames of more than 131072 bytes take part (a smaller frame is what window_log 17 writes); their anchors are
            listed frame by frame in submission order, each frame's in position order.
  hash      gear hash of the 64 bytes ending at p: sum over k < 64 of GEAR[F[p - k]] << k mod 2^64, GEAR[b] = splitmix64(b).
            Positions p >= 63.  (Ending at p, so that a stream chunk needs no byte after it.)
  anchor    p passes when its hash's top 7 bits are 0 (about 1 in 128); p is an anchor when it passes and no position in
            [max(0, p - 15), p) passes: at most one anchor in any 16 positions, whatever the input.
  key       (hash * 0x9E3779B97F4A7C15 mod 2^64) >> 32.
  candidate the anchor listed last before p with the same key (over the whole submission); kept when it is of the same frame and
            p minus its position lies in (131072, 2^window_log].
  block     per 128 KiB block, the anchors in the block in order, each with a candidate offset o: skipped when it lies inside the
            last kept match at offset o; else its 64 bytes must equal those o back (they may start in the previous block).  The
            match runs forward from the anchor up to the block's end, and backward from the window's start down to the largest
            of the block's start, the point where the source would leave the frame, and `maxend`, the end of the last kept
            match (0 at the block's start).  It is kept when 64 or more bytes remain; a kept match that starts at the last
            kept one's end with the same offset joins it.
  forced    in every segment [s, e), the block's kept matches clipped to it, pieces under 5 bytes dropped.  The parse runs as
            it does up to a segment's end up to the next piece's start (lanes q with q + 5 <= that start, matches extended no
            further); the piece is then one sequence with the literals since the last match, and the parse resumes at its end.
            At LAZY the piece's offset enters the segment's repeat offsets as any match taken does.  (cparse._pieces clips the
            matches; both levels' segment loops take the pieces.)
  header    Window_Descriptor exponent min(window_log, max(17, ceil(log2 n))) (Single_Segment 0, mantissa 0; cparse.frame_header).

`parse` is cparse.parse with `forced`'s matches; cparse.reference_frame(..., window_log=) assembles the frame."""
import numpy as np

import cparse

BLOCK, WINDOW = cparse.BLOCK, cparse.WINDOW
LDM_LEN = 64
LDM_MASK_SHIFT = 57
LDM_QUIET = 15
KEY_MUL = 0x9E3779B97F4A7C15
_M = (1 << 64) - 1


def splitmix64(x):
    z = (x + 0x9E3779B97F4A7C15) & _M
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M
    return z ^ (z >> 31)


GEAR = np.array([splitmix64(b) for b in range(256)], dtype=np.uint64)


def gear_hashes(data):
    """The gear hash of the 64 bytes starting at every position p with p + 64 <= len(data), as a uint64 array (the hash of the
    anchor position p + 63)."""
    a = np.frombuffer(bytes(data), dtype=np.uint8)
    m = len(a) - LDM_LEN + 1
    if m <= 0:
        return np.zeros(0, dtype=np.uint64)
    g = GEAR[a]
    h = np.zeros(m, dtype=np.uint64)
    with np.errstate(over="ignore"):
        for k in range(LDM_LEN):
            h += g[k:k + m] << np.uint64(LDM_LEN - 1 - k)
    return h


def anchors(data):
    """(positions, keys) of the anchors of data, in position order."""
    h = gear_hashes(data)
    if not len(h):
        return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.uint64)
    passes = (h >> np.uint64(LDM_MASK_SHIFT)) == 0
    cs = np.concatenate([[0], np.cumsum(passes)])
    p = np.arange(len(h))
    before = cs[p] - cs[np.maximum(p - LDM_QUIET, 0)]      # passing positions in [max(0, p - 15), p)
    pos = np.nonzero(passes & (before == 0))[0]
    with np.errstate(over="ignore"):
        keys = (h[pos] * np.uint64(KEY_MUL)) >> np.uint64(32)
    return pos.astype(np.int64) + LDM_LEN - 1, keys


def candidates(frames, window_log):
    """Per frame, [(position, offset)] of its anchors with a kept candidate (offset > 0), in position order; [] for frames of
    131072 bytes or fewer."""
    last = {}
    out = []
    for fi, f in enumerate(frames):
        got = []
        if len(f) > BLOCK:
            pos, keys = anchors(f)
            for p, k in zip(pos.tolist(), keys.tolist()):
                prev = last.get(k)
                if prev is not None and prev[0] == fi and WINDOW < p - prev[1] <= (1 << window_log):
                    got.append((p, p - prev[1]))
                last[k] = (fi, p)
        out.append(got)
    return out


def block_matches(F, b0, n, cands):
    """The kept matches [(start, length, offset)] (block-relative) of the block F[b0:b0 + n], from the frame's candidates in it."""
    kept = []
    maxend = 0
    for p, off in cands:
        at = p - b0
        if kept and off == kept[-1][2] and at < kept[-1][0] + kept[-1][1]:
            continue
        w0 = p - LDM_LEN + 1
        if F[w0:p + 1] != F[w0 - off:p + 1 - off]:
            continue
        e = at + 1
        while e < n and F[b0 + e] == F[b0 + e - off]:
            e += 1
        lo = max(maxend, off - b0 if off > b0 else 0)
        s = max(w0 - b0, lo)
        while s > lo and F[b0 + s - 1] == F[b0 + s - 1 - off]:
            s -= 1
        if e < s + LDM_LEN:
            continue
        if kept and off == kept[-1][2] and s == kept[-1][0] + kept[-1][1]:
            kept[-1] = (kept[-1][0], e - kept[-1][0], off)
        else:
            kept.append((s, e - s, off))
        maxend = e
    return kept


def forced(frames, window_log):
    """Per frame, per block, the block's kept matches (block_matches)."""
    out = []
    for f, cands in zip(frames, candidates(frames, window_log)):
        F = bytes(f)
        blocks, pos, i = [], 0, 0
        while True:
            n = min(BLOCK, len(F) - pos)
            mine = []
            while i < len(cands) and cands[i][0] < pos + n:
                mine.append(cands[i])
                i += 1
            blocks.append(block_matches(F, pos, n, mine) if mine else [])
            pos += n
            if pos >= len(F):
                break
        out.append(blocks)
    return out


def parse(frames, window_log, content=None, level=cparse.FASTEST):
    """The parse of every frame of one submission at window_log and `level`: the regular parse with the long matches forced
    (none at window_log 17, where no long-match kernel runs)."""
    return cparse.parse(frames, content, level, forced(frames, window_log) if window_log > cparse.WINDOW_LOG_MIN else None)


def offsets(blocks):
    """Every offset of a parse's sequences."""
    return [of for b in blocks if b[0] != "rle" for _, _, of in b[1]]
