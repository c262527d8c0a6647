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
            At LAZY the piece's offset enters the segment's repeat offsets as any match taken does.
  header    Window_Descriptor exponent min(window_log, max(17, ceil(log2 n))) (Single_Segment 0, mantissa 0).

`parse` gives what cparse.parse / clazy.parse give; `reference_frame` assembles the frame."""
import numpy as np

import clazy
import cparse

BLOCK, WINDOW, MIN_MATCH, CM_WARPS = cparse.BLOCK, cparse.WINDOW, cparse.MIN_MATCH, cparse.CM_WARPS
LDM_LEN = 64
LDM_MASK_SHIFT = 57
LDM_QUIET = 15
KEY_MUL = 0x9E3779B97F4A7C15
WINDOW_LOG_MIN, WINDOW_LOG_MAX = 17, 27
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


def frame_window_log(n, window_log):
    """The Window_Descriptor exponent of a frame of n bytes."""
    if window_log <= WINDOW_LOG_MIN:
        return WINDOW_LOG_MIN
    c = WINDOW_LOG_MIN
    while c < window_log and (1 << c) < n:
        c += 1
    return c


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


def _pieces(kept, s, e):
    """The block's kept matches clipped to [s, e): [(cs, ce, off)], pieces under MIN_MATCH bytes dropped."""
    out = []
    for st, ln, off in kept:
        if st >= e:
            break
        cs, ce = max(st, s), min(st + ln, e)
        if ce >= cs + MIN_MATCH:
            out.append((cs, ce, off))
    return out


def _segment_fastest(F, base, n, back, s, e, t1, H14, H12, H17, dic, pieces):
    """cparse._segment with forced pieces."""
    W, CAP = cparse.WINDOW, cparse.CM_CAP
    tp = {}
    for q in range(max(s - cparse.CM_SEED, -min(back, cparse.CM_SEED)), min(s, n - MIN_MATCH + 1)):
        tp[H12[base + q]] = q
    seqs, lits = [], []
    p = anchor = s
    k = 0
    while True:
        ee = pieces[k][0] if k < len(pieces) else e
        last = ee - MIN_MATCH + 1
        while p < last:
            hi = min(p + 32, last)
            found = None
            for q in range(p, hi):
                fq = base + q
                lim = min(CAP, ee - q)
                best = cand = 0
                c1 = t1[H14[fq]]
                if c1 < q:
                    best, cand = cparse._mlen(F, fq, F, base + c1, lim), q - c1
                c2 = tp.get(H12[fq])
                if c2 is not None and c2 < q and q - c2 <= W:
                    l2 = cparse._mlen(F, fq, F, base + c2, lim)
                    if l2 > best or (l2 == best and q - c2 < cand):
                        best, cand = l2, q - c2
                xlim = ee - q
                if dic is not None and back + q < W:
                    d = dic.tab.get(H17[fq])
                    if d is not None and back + q + dic.n - d <= W:
                        off3, rest = back + q + dic.n - d, dic.n - d
                        l3 = cparse._mlen(F, fq, dic.data, d, min(lim, rest))
                        if l3 > best or (l3 == best and off3 < cand):
                            best, cand, xlim = l3, off3, min(xlim, rest)
                if best >= MIN_MATCH:
                    found = (q, best, cand, xlim)
                    break
            for q in range(p, hi):
                h = H12[base + q]
                if tp.get(h, -W - 1) < q:
                    tp[h] = q
            if found is None:
                p += 32
                continue
            q, ml, off, xlim = found
            if ml == CAP:
                fq = base + q
                if off > back + q:
                    ref, r0 = dic.data, dic.n - (off - (back + q))
                else:
                    ref, r0 = F, fq - off
                while ml < xlim and F[fq + ml] == ref[r0 + ml]:
                    ml += 1
            lits.append(F[base + anchor:base + q])
            seqs.append((q - anchor, ml, off))
            anchor = p = q + ml
        if k == len(pieces):
            break
        cs, ce, off = pieces[k]
        lits.append(F[base + anchor:base + cs])
        seqs.append((cs - anchor, ce - cs, off))
        anchor = p = ce
        k += 1
    lits.append(F[base + anchor:base + e])
    return b"".join(lits), seqs, e - anchor


def _segment_lazy(F, base, n, back, s, e, t1, H14, H11, H17, dic, pieces):
    """clazy._segment with forced pieces."""
    tab = {}

    def insert(q):
        h = H11[base + q]
        b = tab.get(h)
        if b is None:
            tab[h] = [q]
        else:
            b.insert(0, q)
            del b[clazy.LZ_WAYS:]

    for q in range(max(s - clazy.LZ_SEED, -back), min(s, n - MIN_MATCH + 1)):
        insert(q)
    reps = []
    seqs, lits = [], []
    p = anchor = s
    k = 0

    def take(off):
        if off in reps:
            reps.remove(off)
        reps.insert(0, off)
        del reps[3:]

    def lane(q, ee):
        fq = base + q
        lim = min(clazy.LZ_CAP, ee - q)
        best = None
        for o in reps:
            if o <= back + q and o <= WINDOW:
                ml = clazy._mlen(F, fq, F, fq - o, lim)
                if ml >= MIN_MATCH and (best is None or 4 * ml > best[0]):
                    best = (4 * ml, ml, o, ee - q)
        cands = []
        c1 = t1[H14[fq]]
        if c1 < q:
            cands.append(c1)
        cands += [c for c in tab.get(H11[fq], ()) if c < q]
        for c in cands:
            o = q - c
            ml = clazy._mlen(F, fq, F, fq - o, lim)
            if ml >= MIN_MATCH:
                g = 4 * ml - clazy._cost(o, False)
                if best is None or g > best[0]:
                    best = (g, ml, o, ee - q)
        if dic is not None and back + q < WINDOW:
            d = dic.tab.get(H17[fq])
            if d is not None and back + q + dic.n - d <= WINDOW:
                o, rest = back + q + dic.n - d, dic.n - d
                ml = clazy._mlen(F, fq, dic.data, d, min(lim, rest))
                if ml >= MIN_MATCH:
                    g = 4 * ml - clazy._cost(o, False)
                    if best is None or g > best[0]:
                        best = (g, ml, o, min(ee - q, rest))
        return best

    while True:
        ee = pieces[k][0] if k < len(pieces) else e
        last = ee - MIN_MATCH + 1
        while p < last:
            hi = min(p + 32, last)
            found = None
            for q in range(p, hi):
                c = lane(q, ee)
                if c is not None:
                    found = (q, c)
                    break
            if found is not None:
                j = found[0]
                score = found[1][0]
                for q in range(j + 1, min(j + clazy.LZ_DEPTH + 1, hi)):
                    c = lane(q, ee)
                    if c is not None and c[0] - clazy.LZ_LANE_COST * (q - j) > score:
                        found, score = (q, c), c[0] - clazy.LZ_LANE_COST * (q - j)
            for q in range(p, hi):
                insert(q)
            if found is None:
                p += 32
                continue
            q, (_, ml, off, xlim) = found
            if ml == clazy.LZ_CAP:
                fq = base + q
                if off > back + q:
                    ref, r0 = dic.data, dic.n - (off - (back + q))
                else:
                    ref, r0 = F, fq - off
                while ml < xlim and F[fq + ml] == ref[r0 + ml]:
                    ml += 1
            lits.append(F[base + anchor:base + q])
            seqs.append((q - anchor, ml, off))
            take(off)
            anchor = p = q + ml
        if k == len(pieces):
            break
        cs, ce, off = pieces[k]
        lits.append(F[base + anchor:base + cs])
        seqs.append((cs - anchor, ce - cs, off))
        take(off)
        anchor = p = ce
        k += 1
    lits.append(F[base + anchor:base + e])
    return b"".join(lits), seqs, e - anchor


def _parse_block(F, base, n, back, H_t1, H_tab, H17, dic, kept, lazy):
    if not kept:
        return (clazy if lazy else cparse).parse_block(F, base, n, back, H_t1, H_tab, H17, dic)
    blk = F[base:base + n]
    if blk.count(blk[:1]) == n:
        return ("rle", blk[0], n)
    t1 = [BLOCK] * (1 << (clazy.LZ_T1_LOG if lazy else cparse.CM_T1_LOG))
    for q in range(n - MIN_MATCH, -1, -1):
        t1[H_t1[base + q]] = q
    seglen = -(-n // CM_WARPS)
    lits, seqs, carry = [], [], 0
    seg = _segment_lazy if lazy else _segment_fastest
    for w in range(CM_WARPS):
        s = min(n, w * seglen)
        e = min(n, s + seglen)
        sl, ss, trail = seg(F, base, n, back, s, e, t1, H_t1, H_tab, H17, dic, _pieces(kept, s, e))
        lits.append(sl)
        if ss:
            ss[0] = (ss[0][0] + carry, ss[0][1], ss[0][2])
            carry = trail
        else:
            carry += trail
        seqs += ss
    return (b"".join(lits), seqs)


def parse_frame(data, kept_blocks, dic=None, lazy=False):
    """The blocks of one frame with its forced matches (one list per block, from `forced`)."""
    F = bytes(data)
    if lazy:
        H_t1, H_tab = cparse.hashes(F, clazy.LZ_T1_LOG), cparse.hashes(F, clazy.LZ_TAB_LOG)
    else:
        H_t1, H_tab = cparse.hashes(F, cparse.CM_T1_LOG), cparse.hashes(F, cparse.CM_TP_LOG)
    H17 = cparse.hashes(F[:WINDOW + 4], cparse.CD_LOG) if dic is not None else None
    out, pos, k = [], 0, 0
    while True:
        n = min(BLOCK, len(F) - pos)
        out.append(_parse_block(F, pos, n, min(pos, WINDOW), H_t1, H_tab, H17, dic, kept_blocks[k], lazy))
        pos += n
        k += 1
        if pos >= len(F):
            return out


def parse(frames, window_log, content=None, lazy=False):
    """The parse of every frame of one submission at window_log (Fastest, or LAZY with lazy=True)."""
    dic = cparse.match_dict(content)
    return [parse_frame(f, kb, dic, lazy) for f, kb in zip(frames, forced(frames, window_log))]


def reference_frame(data, blocks, window_log, checksum=True, dict_id=0, dict_tables=None, lazy=False):
    """The frame for `data` whose parse is `blocks`, with the Window_Descriptor of window_log."""
    if lazy:
        out = clazy.reference_frame(data, blocks, checksum, dict_id, dict_tables)
    else:
        out = cparse.reference_frame(data, blocks, checksum, dict_id, dict_tables)
    return out[:5] + bytes([(frame_window_log(len(data), window_log) - 10) << 3]) + out[6:]


def offsets(blocks):
    """Every offset of a parse's sequences."""
    return [of for b in blocks if b[0] != "rle" for _, _, of in b[1]]
