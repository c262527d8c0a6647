"""The compressor's LAZY level (an extension) written out plainly: what k_cmatch<DICT, true> must produce for every block, the
repeat-offset pass k_cenc<TABLES, true> runs before encoding, and the frame the compressor must write.

This module restates the rules of zstd-rs_b200/csrc/compress.cu at B200Z_LEVEL_LAZY and DESIGN.md section 4.4 in Python, calling
nothing in the library.  It shares the Fastest model's hashing, dictionary table, block and frame drivers, XXH64 and headers
(tests/cparse.py): `LAZY` is the level cparse.parse and cparse.reference_frame take.  The parse is per block ("rle", byte, n) or
(literals, [(ll, ml, of), ...]) with `of` the actual offset, and `reps` turns a block's sequences into the records the encoder
codes: `of` is then Offset_Value - 3 (mod 2^32).  The rules beyond the
Fastest parse's blocks, t1, segments, dictionary and packing:

  t1        as Fastest's, over hash5(p, 15).
  table     per segment, a table of the K = 6 most recent positions per hash5(p, 10), newest first.  It is seeded, in position
            order, with every q in [max(s - 32768, -back), s) with q + 5 <= n, then every round inserts its valid lanes in
            position order.  (The kernel stores q - (s - 32768) as a u16, below 49152; 0xffff marks an empty way.)  An entry
            counts when it is < q (a round's lanes past the chosen match are inserted too).
  reps      per segment, the three most recent distinct offsets of the matches it took, newest first, empty at its start.
            Taking offset o moves o to the front (removing it if present; else the oldest drops out).
  lanes     every lane q of [p, p + 32) with q + 5 <= e verifies, for up to min(32, e - q) bytes, in this order: the reps
            (rep0, rep1, rep2: each when set, o <= back + q and o <= 131072, so the source lies in the frame and the window),
            t1 (when c1 < q), the table's entries newest first, and the dictionary (as Fastest).  A candidate scores
            gain = 4 * ml - cost with cost 0 for a rep and floor(log2(o)) otherwise; only ml >= 5 counts; a strictly higher gain
            replaces the lane's best, so a tie keeps the earlier candidate.
  choice    j is the first lane with a match.  Lanes j + d, d = 0 .. D (D = 4), inside the round and with a match, score
            gain - 3 d; the highest score wins, a tie going to the earlier lane.  The winner's literals run from the anchor to its lane; a match of
            exactly 32 bytes is extended to e (or to the dictionary's end).  The next round starts at the match's end; every
            valid lane of the round is inserted into the table, whichever lane won.
  rep pass  per Compressed block, over its packed sequences in order, the decoder's offset history (RFC 8878 3.1.2.5) with three
            unknown slots at the block's start.  LL > 0: the first known slot of rep0, rep1, rep2 equal to the offset gives
            Offset_Value 1, 2, 3.  LL = 0: rep1 -> 1, rep2 -> 2, rep0 - 1 -> 3 (first that is known and equal).  Any other
            sequence is coded raw (o + 3).  The history then moves as the decoder moves it; unknown slots move like known ones.

`cases()` builds the crafted inputs; each case's id names the rule it sits on."""
import random

import cparse

BLOCK, WINDOW, MIN_MATCH, CM_WARPS = cparse.BLOCK, cparse.WINDOW, cparse.MIN_MATCH, cparse.CM_WARPS
LZ_T1_LOG = 15           # t1, the block's first occurrences (Fastest: 14)
LZ_TAB_LOG = 10          # buckets of a segment's table
LZ_WAYS = 6              # K: positions per bucket
LZ_SEED = 32768          # bytes before its segment a segment's table is seeded from
LZ_CAP = 32              # bytes a lane verifies before the chosen match is extended
LZ_DEPTH = 4             # D: lanes after the first match that compete with it
LZ_LANE_COST = 3         # gain a later lane gives up per byte it starts later
CSEG_SEQS = cparse.CSEG_SEQS


def _cost(o, rep):
    return 0 if rep else o.bit_length() - 1


def _segment(F, base, n, back, s, e, t1, H15, H10, H17, dic, pieces):
    """Parse of segment [s, e) of the block at F[base:base + n] with its forced pieces [(cs, ce, off)] (empty: none): (literals,
    sequences, trailing literal count)."""
    tab = {}

    def insert(q):
        h = H10[base + q]
        b = tab.get(h)
        if b is None:
            tab[h] = [q]
        else:
            b.insert(0, q)
            del b[LZ_WAYS:]

    for q in range(max(s - LZ_SEED, -back), min(s, n - MIN_MATCH + 1)):
        insert(q)
    reps = []
    seqs, lits = [], []
    p = anchor = s

    def take(off):
        if off in reps:
            reps.remove(off)
        reps.insert(0, off)
        del reps[3:]

    def lane(q, stop):
        """The lane's best candidate (gain, ml, off, xlim), or None."""
        fq = base + q
        lim = min(LZ_CAP, stop - q)
        best = None
        for o in reps:
            if o <= back + q and o <= WINDOW:
                ml = cparse._mlen(F, fq, F, fq - o, lim)
                if ml >= MIN_MATCH and (best is None or 4 * ml > best[0]):
                    best = (4 * ml, ml, o, stop - q)
        cands = []
        c1 = t1[H15[fq]]
        if c1 < q:
            cands.append(c1)
        cands += [c for c in tab.get(H10[fq], ()) if c < q]
        for c in cands:
            o = q - c
            ml = cparse._mlen(F, fq, F, fq - o, lim)
            if ml >= MIN_MATCH:
                g = 4 * ml - _cost(o, False)
                if best is None or g > best[0]:
                    best = (g, ml, o, stop - q)
        if dic is not None and back + q < WINDOW:
            d = dic.tab.get(H17[fq])
            if d is not None and back + q + dic.n - d <= WINDOW:
                o, rest = back + q + dic.n - d, dic.n - d
                ml = cparse._mlen(F, fq, dic.data, d, min(lim, rest))
                if ml >= MIN_MATCH:
                    g = 4 * ml - _cost(o, False)
                    if best is None or g > best[0]:
                        best = (g, ml, o, min(stop - q, rest))
        return best

    for k in range(len(pieces) + 1):
        stop = pieces[k][0] if k < len(pieces) else e   # the parse runs up to the next piece's start
        last = stop - MIN_MATCH + 1             # lanes q < last have q + 5 <= stop
        while p < last:
            hi = min(p + 32, last)
            found = None
            for q in range(p, hi):
                c = lane(q, stop)
                if c is not None:
                    found = (q, c)
                    break
            if found is not None:
                j = found[0]
                score = found[1][0]
                for q in range(j + 1, min(j + LZ_DEPTH + 1, hi)):
                    c = lane(q, stop)
                    if c is not None and c[0] - LZ_LANE_COST * (q - j) > score:
                        found, score = (q, c), c[0] - LZ_LANE_COST * (q - j)
            for q in range(p, hi):              # every valid lane inserts, before or after the chosen one
                insert(q)
            if found is None:
                p += 32
                continue
            q, (_, ml, off, xlim) = found
            if ml == LZ_CAP:
                fq = base + q
                if off > back + q:              # the source lies in the dictionary: stop at its end
                    ref, r0 = dic.data, dic.n - (off - (back + q))
                else:
                    ref, r0 = F, fq - off
                while ml < xlim and F[fq + ml] == ref[r0 + ml]:
                    ml += 1
            lits.append(F[base + anchor:base + q])
            seqs.append((q - anchor, ml, off))
            take(off)
            anchor = p = q + ml
        if k < len(pieces):                     # the piece is one sequence and a repeat offset; the parse resumes at its end
            cs, ce, off = pieces[k]
            lits.append(F[base + anchor:base + cs])
            seqs.append((cs - anchor, ce - cs, off))
            take(off)
            anchor = p = ce
    lits.append(F[base + anchor:base + e])
    assert len(seqs) <= CSEG_SEQS
    return b"".join(lits), seqs, e - anchor


def reps(seqs):
    """The rep pass over one block's sequences: [(ll, ml, Offset_Value), ...] (1-3 repeat codes, o + 3 raw)."""
    h = [None, None, None]                      # rep0, rep1, rep2; None: unknown
    out = []
    for ll, ml, o in seqs:
        if ll > 0:
            names = [(1, h[0]), (2, h[1]), (3, h[2])]
        else:
            names = [(1, h[1]), (2, h[2]), (3, None if h[0] is None else h[0] - 1)]
        ov = next((v for v, x in names if x is not None and x == o), o + 3)
        out.append((ll, ml, ov))
        if ov > 3:
            h = [o, h[0], h[1]]
        else:
            r = ov - 1 + (1 if ll == 0 else 0)
            if r == 1:
                h = [h[1], h[0], h[2]]
            elif r == 2:
                h = [h[2], h[0], h[1]]
            elif r == 3:
                h = [o, h[0], h[1]]
    return out


def records(seqs):
    """What k_cenc<TABLES, true> hands encode_block: (ll, ml, Offset_Value - 3 mod 2^32)."""
    return [(ll, ml, (ov - 3) & 0xFFFFFFFF) for ll, ml, ov in reps(seqs)]


LAZY = cparse.Level(LZ_T1_LOG, LZ_TAB_LOG, _segment, records)


# ---------------------------------------------------------------------------------------------------------------------------
# the crafted cases
# ---------------------------------------------------------------------------------------------------------------------------
Case, rand, plant, seg_bounds = cparse.Case, cparse.rand, cparse.plant, cparse.seg_bounds


def keep_in_table(buf, first, dst, protect):
    """Changes bytes of buf so that no position in (first, dst) shares position first's bucket with other bytes: its entry is then
    still in the table when the lane at dst looks it up.  Bytes in `protect` are left alone."""
    target = cparse.hash5(buf, first, LZ_TAB_LOG)
    while True:
        bad = [p for p in range(first + 1, dst)
               if cparse.hash5(buf, p, LZ_TAB_LOG) == target and buf[p:p + 5] != buf[first:first + 5]]
        if not bad:
            return
        for p in bad:
            i = next(i for i in range(p, p + 5) if i not in protect)
            buf[i] ^= 0x3C


def choice(rng):
    """Lazy choice: a 5-byte match at lane z and a 30-byte one at z + 1 (z + 1 wins); an 8-byte match at z (offset 5000, cost 12)
    against a 9-byte one at z + 1 (offset 9000, cost 13): scores 32 - 12 and 36 - 13 - 3 tie, so z is kept.  The sources lie in
    earlier segments than the targets (40000-byte blocks, seglen 5000), which sit at lane 3 of a round."""
    out = []
    s1 = seg_bounds(40000, 1)[0]
    z = s1 + 32 * 40 + 3
    buf = rand(rng, 40000)
    plant(buf, z + 1, 1000, 30)
    buf[2000:2005] = buf[z:z + 5]               # a 5-byte source for lane z
    buf[2005] = buf[z + 5] ^ 0x11
    keep_in_table(buf, 2000, z, set(range(1999, 2006)) | set(range(999, 1031)) | set(range(z - 1, z + 32)))
    out.append(Case("lazy", "later-lane-wins", [buf]))
    buf = rand(rng, 40000)
    z = seg_bounds(40000, 3)[0] + 32 * 40 + 3
    t = bytes(buf[z:z + 10])
    y, x = z - 5000, z + 1 - 9000
    buf[y:y + 8] = t[:8]
    buf[y + 8] = t[8] ^ 0x21
    buf[x:x + 9] = t[1:10]
    buf[x + 9] = buf[z + 10] ^ 0x42
    protect = set(range(y - 1, y + 9)) | set(range(x - 1, x + 10)) | set(range(z - 1, z + 11))
    keep_in_table(buf, y, z, protect)
    keep_in_table(buf, x, z + 1, protect)
    out.append(Case("lazy", "tie-keeps-first-lane", [buf]))
    return out


def repeats(rng):
    """A repeat candidate where t1 and the table miss: in segment 4 a 20-byte match at offset 68000 (through t1), then 500 bytes
    later 20 bytes from 68000 back again, whose source's t1 entry is an earlier 5-byte decoy and which is older than the table's
    seeds.  A 64-byte repeat across a segment start: the next segment's first match has LL 0 and rep0's offset (coded raw).
    A block whose first match repeats the previous block's last offset (coded raw: the history starts unknown)."""
    out = []
    buf = rand(rng, BLOCK)
    plant(buf, 70000, 2000, 20)
    plant(buf, 70500, 2500, 20)
    buf[100:105] = buf[2500:2505]
    buf[105] = buf[2505] ^ 0x77
    out.append(Case("rep", "found-where-t1-and-table-miss", [buf]))
    buf = rand(rng, BLOCK)
    s = seg_bounds(BLOCK, 3)[0]
    plant(buf, s - 32, s - 300, 64)
    keep_in_table(buf, s - 268, s, set(range(s - 301, s - 235)) | set(range(s - 33, s + 33)))
    out.append(Case("rep", "ll0-rep0-across-segment-start", [buf]))
    buf = rand(rng, 2 * BLOCK)
    plant(buf, BLOCK - 200, BLOCK - 1200, 20)
    plant(buf, BLOCK + 500, BLOCK - 500, 20)
    out.append(Case("rep", "block-starts-with-previous-blocks-offset", [buf]))
    return out


def buckets(rng):
    """K-way overflow: a source in the previous block (t1 cannot see it), then K (evicted) or K - 1 (kept) positions of its
    bucket before the 20-byte copy in segment 0 of the second block."""
    out = []
    for extra, name in ((LZ_WAYS, "K-newer-evict"), (LZ_WAYS - 1, "K-1-newer-keep")):
        buf = rand(rng, 2 * BLOCK)
        a, z = BLOCK - 1000, BLOCK + 3000
        plant(buf, z, a, 20)
        protect = set(range(a - 1, a + 21)) | set(range(z - 1, z + 21))
        keep_in_table(buf, a, z, protect)
        target = cparse.hash5(buf, a, LZ_TAB_LOG)
        at = BLOCK + 500
        for _ in range(extra):                  # 5 random bytes with the source's bucket, 100 bytes apart
            while True:
                cand = bytes(rng.getrandbits(8) for _ in range(5))
                tmp = bytearray(cand)
                if cparse.hash5(tmp, 0, LZ_TAB_LOG) == target:
                    break
            buf[at:at + 5] = cand
            at += 100
        out.append(Case("bucket", name, [buf]))
    return out


def seeds(rng):
    """A source exactly LZ_SEED bytes before segment 0 of the last block (the oldest seed) and LZ_SEED + 1 (not seeded; its second
    position is), no position in between sharing their buckets; t1 cannot see the previous block."""
    out = []
    for d in (LZ_SEED, LZ_SEED + 1):
        buf = rand(rng, 2 * BLOCK)
        b = BLOCK
        plant(buf, b + 2000, b - d, 24)
        protect = set(range(b - d - 1, b - d + 25)) | set(range(b + 1999, b + 2025))
        keep_in_table(buf, b - LZ_SEED, b + 2000, protect)
        keep_in_table(buf, b - d + 1, b + 2001, protect)
        out.append(Case("seed", f"source-{d}-before-segment" + ("=LZ_SEED" if d == LZ_SEED else "=LZ_SEED+1"), [buf]))
    return out


def dictionaries(rng):
    """The Fastest model's dictionary cases, and a repeat whose source would lie before the frame: a dictionary match at offset
    o, then 40 bytes later the dictionary's bytes continue at the same distance.  The rep candidate must not count (its source
    lies in the dictionary), so the match takes the dictionary table's later copy."""
    out = [Case("dict", c.id.split("-", 1)[1], c.frames, c.content) for c in cparse.cases("dict")]
    content = rand(rng, 3000)
    f = rand(rng, 3000)
    content[2500:2520] = content[1060:1080]     # the dictionary's table finds the later copy
    plant(f, 100, 1000, 20, content)
    plant(f, 160, 1060, 20, content)
    out.append(Case("dict", "rep-source-before-frame", [f], content))
    return out


def realistic():
    return [Case("data", c.id.split("-", 1)[1], c.frames, c.content) for c in cparse.cases("data")]


GROUPS = {"lazy": choice, "rep": repeats, "bucket": buckets, "seed": seeds, "dict": dictionaries}


def cases(group=None):
    """The crafted cases (all groups, or one), built from fixed seeds, plus the Fastest model's shapes and the realistic group."""
    out = []
    for i, (g, fn) in enumerate(GROUPS.items()):
        if group is None or g == group:
            out += fn(random.Random(0x1A2F + i))
    if group is None or group == "shape":
        out += [Case("shape", c.id.split("-", 1)[1], c.frames, c.content) for c in cparse.cases("shape")]
    if group is None or group == "data":
        out += realistic()
    return out
