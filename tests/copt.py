"""The compressor's OPT level (an extension) written out plainly: what k_copt<DICT, LONG> must produce for every block.

This module restates the rules of zstd-rs_b200/csrc/compress.cu at B200Z_LEVEL_OPT and DESIGN.md section 4.4 in Python, calling
nothing in the library.  It shares the Fastest model's blocks, segments, dictionary table, packing, block and frame drivers, XXH64
and headers (tests/cparse.py), and LAZY's repeat-offset pass (tests/clazy.py `records`): `OPT` is the level cparse.parse and
cparse.reference_frame take.  The parse is per block ("rle", byte, n) or (literals, [(ll, ml, of), ...]) with `of` the actual
offset.  The rules beyond the Fastest parse's blocks, segments, dictionary and packing:

  chain     hash(q) = hash5(q, 13) over the frame.  prev(q) is the nearest earlier position of the same frame with the same hash
            (none before the frame's first byte).  Only positions with q + 5 <= the frame's length are hashed.
  finder    position q of segment [s, e) whose part (the range up to the next forced piece, or e) ends at `stop`, with q + 5 <=
            stop, walks c = prev(q), prev(prev(q)), ... while q - c <= 131072, visiting at most D = 24 entries (collisions
            count).  Each entry is verified for up to min(CAP, stop - q) bytes (CAP = 32); one longer than every earlier one (and
            >= 5) is a candidate, the shortest dropped when there are more than M = 4; the walk ends when a verification reaches
            its limit.  With a dictionary and back + q < 131072, the dictionary table's entry (as Fastest) is verified for
            min(CAP, stop - q, the bytes to the dictionary's end) and appended the same way.  The list depends on the input only.
  prices    integers in 1/256 bit.  L(x) = 256 * floor(log2 x) + the 8 bits after x's leading one (a linear mantissa).  A literal
            byte b costs L(n) - L(count of b in the block's n bytes).  A match costs MATCH_W = 1024 plus, for offset o from the
            finder, 256 * floor(log2(o + 3)) + OF_W (OF_W = 512), or REP_W[k] = 256 (k + 1) when it is the node's repeat k.
  reps      per path, the three most recent distinct offsets, newest first, empty at the segment's start; a match with offset o
            moves o to the front (LAZY's rule; forced pieces too).
  dp        from a start a with the segment's current reps, a forward pass over the nodes a, a + 1, ...  Node a costs 0.  At node
            i (its cost now final; i < stop):
              - its repeats are verified when i + 5 <= stop: rep k when set, o <= back + i and o <= 131072, for min(CAP, stop - i)
                bytes;
              - if a repeat or a finder candidate has >= SUFF = CAP bytes, the longest (the first in the order rep0, rep1, rep2,
                finder list on a tie) is taken at once: the DP closes at i, and the match, extended to `stop` (a dictionary match
                to the dictionary's end too), follows the path; the next DP starts after it;
              - else i relaxes i + 1 with its literal, then every length l in [5, SUFF): the offers are each repeat verified
                for >= l bytes (REP_W[k]) and the first finder candidate with >= l bytes; the cheapest offer, the first in the
                order rep0, rep1, rep2, finder on a tie, replaces node i + l's path when strictly cheaper.
            The DP closes at node stop, or at node a + W (W = 256) when that is before stop; the next DP starts there with that
            node's reps.  Closing emits the path to the node (its literals join the next sequence).
  long      forced pieces end their part: the DP closes at the piece's start, the piece is one sequence and a repeat.

`cases()` builds the crafted inputs; each case's id names the rule it sits on."""
import functools
import random

import numpy as np

import clazy
import cparse

BLOCK, WINDOW, MIN_MATCH, CM_WARPS = cparse.BLOCK, cparse.WINDOW, cparse.MIN_MATCH, cparse.CM_WARPS
CSEG_SEQS = cparse.CSEG_SEQS
OPT_HASH_LOG = 13        # H: the chain's hash
OPT_DEPTH = 24           # D: chain entries a position visits
OPT_CANDS = 4            # M: candidates kept per position
OPT_CAP = 32             # CAP: bytes a candidate is verified for; also SUFF, the length taken at once
OPT_SUFF = OPT_CAP
OPT_WIN = 256            # W: nodes a DP spans before it closes
# prices, in 1/256 bit
MATCH_W = 256 * 4        # any match (lengths below SUFF have no ML extra bits)
OF_W = 256 * 2           # an offset code, beyond its bits
REP_W = (256 * 1, 256 * 2, 256 * 3)   # a repeat, by its index
INF = 1 << 30


def log2fp(x):
    """L(x), x >= 1: 256 * floor(log2 x) + the 8 bits after x's leading one."""
    k = x.bit_length() - 1
    m = (x << 8 >> k) & 255 if k <= 8 else (x >> (k - 8)) & 255
    return 256 * k + m


def of_price(o):
    return 256 * ((o + 3).bit_length() - 1) + OF_W


def lit_prices(blk):
    """Per byte value, the price of one literal in a block whose bytes are blk."""
    cnt = np.bincount(np.frombuffer(bytes(blk), dtype=np.uint8), minlength=256).tolist()
    ln = log2fp(len(blk))
    return [ln - log2fp(c) if c else INF for c in cnt]


def chain(H):
    """prev over a frame's hash list H: the nearest earlier position with the same hash, or -1."""
    h = np.asarray(H, dtype=np.int64)
    prev = np.full(len(h), -1, dtype=np.int64)
    if len(h):
        order = np.argsort(h, kind="stable")
        same = h[order[1:]] == h[order[:-1]]
        prev[order[1:][same]] = order[:-1][same]
    return prev.tolist()


_chain_memo = [None, None]


def _prev(H):
    if _chain_memo[0] is not H:
        _chain_memo[0], _chain_memo[1] = H, chain(H)
    return _chain_memo[1]


def candidates(F, base, back, q, stop, prev, H17, dic):
    """The finder's list at block position q of the block at F[base:]: [(length, offset, extension limit)], lengths increasing."""
    fq = base + q
    lim = min(OPT_CAP, stop - q)
    out, best = [], MIN_MATCH - 1
    c, seen = prev[fq], 0
    while c >= 0 and fq - c <= WINDOW and seen < OPT_DEPTH:
        seen += 1
        ln = cparse._mlen(F, fq, F, c, lim)
        if ln > best:
            out.append((ln, fq - c, stop - q))
            best = ln
            if len(out) > OPT_CANDS:
                del out[0]
            if ln == lim:
                break
        c = prev[c]
    if dic is not None and back + q < WINDOW:
        d = dic.tab.get(H17[fq])
        if d is not None and back + q + dic.n - d <= WINDOW:
            o, rest = back + q + dic.n - d, dic.n - d
            ln = cparse._mlen(F, fq, dic.data, d, min(lim, rest))
            if ln > best:
                out.append((ln, o, min(stop - q, rest)))
                if len(out) > OPT_CANDS:
                    del out[0]
    return out


def push(reps, o):
    """The reps after a match with offset o."""
    return (o,) + tuple(x for x in reps if x != o)[:2]


def dp(F, base, back, a, stop, reps, cands, lit, use_reps=True):
    """One DP from node a with reps: (end node, [(pos, ml, off, xlim) of the path's matches], end reps, taken) where taken is the
    match (pos, ml, off, xlim) taken at once at the end node (ml not yet extended), or None; cands(i) is the finder's list."""
    end = min(stop, a + OPT_WIN)
    size = end - a + OPT_SUFF + 1
    cost = [INF] * size
    bp = [None] * size                          # (from, ml, off, xlim); ml 0: a literal
    rp = [None] * size
    cost[0], rp[0] = 0, tuple(reps)
    taken = None
    i = a
    while True:
        if i == end:
            break
        k = i - a
        ci, ri = cost[k], rp[k]
        fq = base + i
        rl = []                                 # (length, k, off) of the verified repeats
        cl = []
        if i + MIN_MATCH <= stop:
            lim = min(OPT_CAP, stop - i)
            if use_reps:
                for j, o in enumerate(ri):
                    if o <= back + i and o <= WINDOW:
                        ln = cparse._mlen(F, fq, F, fq - o, lim)
                        if ln >= MIN_MATCH:
                            rl.append((ln, j, o))
            cl = cands(i)
            top = None
            for ln, j, o in rl:
                if ln >= OPT_SUFF and (top is None or ln > top[1]):
                    top = (i, ln, o, stop - i)
            if cl and cl[-1][0] >= OPT_SUFF and (top is None or cl[-1][0] > top[1]):
                top = (i, cl[-1][0], cl[-1][1], cl[-1][2])
            if top is not None:
                taken = top
                end = i
                break
        c = ci + lit[F[fq]]
        if c < cost[k + 1]:
            cost[k + 1], bp[k + 1], rp[k + 1] = c, (k, 0, 0), ri
        mx = max([x[0] for x in rl] + [x[0] for x in cl[-1:]] + [0])
        ci_ = 0
        for ln in range(MIN_MATCH, mx + 1):
            mp = MATCH_W
            best = None
            for rln, j, o in rl:
                if rln >= ln:
                    p = REP_W[j]
                    if best is None or p < best[0]:
                        best = (p, o)
            while ci_ < len(cl) and cl[ci_][0] < ln:
                ci_ += 1
            if ci_ < len(cl):
                p = of_price(cl[ci_][1])
                if best is None or p < best[0]:
                    best = (p, cl[ci_][1])
            if best is None:
                continue
            c = ci + mp + best[0]
            t = k + ln
            if c < cost[t]:
                cost[t], bp[t], rp[t] = c, (k, ln, best[1]), push(ri, best[1])
        i += 1
    path = []
    k = end - a
    while k:
        f, ln, o = bp[k]
        if ln:
            path.append((a + f, ln, o))
        k = f
    path.reverse()
    return end, path, rp[end - a], taken, cost[end - a]


def _segment(F, base, n, back, s, e, t1, H13, _H13, H17, dic, pieces, use_reps=True):
    """Parse of segment [s, e) of the block at F[base:base + n] with its forced pieces [(cs, ce, off)]: (literals, sequences,
    trailing literal count)."""
    prev = _prev(H13)
    lit = lit_prices(F[base:base + n])
    seqs, lits = [], []
    reps = ()
    p = anchor = s

    def emit(q, ml, off):
        nonlocal anchor
        lits.append(F[base + anchor:base + q])
        seqs.append((q - anchor, ml, off))
        anchor = q + ml

    for k in range(len(pieces) + 1):
        stop = pieces[k][0] if k < len(pieces) else e
        memo = {}

        def cands(i):
            if i not in memo:
                memo[i] = candidates(F, base, back, i, stop, prev, H17, dic)
            return memo[i]

        while p < stop:
            end, path, r, taken, _ = dp(F, base, back, p, stop, reps, cands, lit, use_reps)
            for q, ml, off in path:
                emit(q, ml, off)
            reps = r
            p = end
            if taken is not None:
                q, ml, off, xlim = taken
                fq = base + q
                if off > back + q:              # the source lies in the dictionary: stop at its end
                    ref, r0 = dic.data, dic.n - (off - (back + q))
                else:
                    ref, r0 = F, fq - off
                while ml < xlim and F[fq + ml] == ref[r0 + ml]:
                    ml += 1
                emit(q, ml, off)
                reps = push(reps, off)
                p = q + ml
        if k < len(pieces):
            cs, ce, off = pieces[k]
            emit(cs, ce - cs, off)
            reps = push(reps, off)
            p = ce
    lits.append(F[base + anchor:base + e])
    assert len(seqs) <= CSEG_SEQS
    return b"".join(lits), seqs, e - anchor


OPT = cparse.Level(OPT_HASH_LOG, OPT_HASH_LOG, _segment, clazy.records)
OPT_NO_REPS = cparse.Level(OPT_HASH_LOG, OPT_HASH_LOG, functools.partial(_segment, use_reps=False), clazy.records)   # model only


# ---------------------------------------------------------------------------------------------------------------------------
# the crafted cases
# ---------------------------------------------------------------------------------------------------------------------------
Case, rand, plant, seg_bounds = cparse.Case, cparse.rand, cparse.plant, cparse.seg_bounds


def suff(rng):
    """A repeat of SUFF - 1 bytes (priced among the others) and one of SUFF bytes (taken at once, then extended to 60), each
    from 3000 bytes back, in segment 1 of a 40000-byte block."""
    out = []
    for n, name in ((OPT_SUFF - 1, "SUFF-1"), (OPT_SUFF, "SUFF"), (60, "SUFF-extended-to-60")):
        buf = rand(rng, 40000)
        s = seg_bounds(40000, 1)[0]
        plant(buf, s + 700, s - 2300, n)
        out.append(Case("suff", f"ml{n}={name}", [buf]))
    return out


def window_cap(rng):
    """Short matches every 7 bytes over more than W positions: the DP closes at a + W, a match that would cross it is cut
    there; and a path through W nodes of literals only."""
    buf = rand(rng, 20000)
    src = bytes(buf[:4000])
    for dst in range(6000, 6000 + 3 * OPT_WIN, 7):
        k = rng.randrange(0, 3900)
        buf[dst:dst + 6] = src[k:k + 6]
    return [Case("wincap", f"matches-across-W={OPT_WIN}", [buf]),
            Case("wincap", "literals-only-W", [rand(rng, 3 * OPT_WIN + 11)])]


def repeats(rng):
    """A repeat that exists only along one path: 9 bytes at offset 777, then 12 literal bytes, then the same offset again; and a
    cost tie: the same 12 bytes at offsets 1000 and 1012, whose codes cost the same."""
    out = []
    buf = rand(rng, 30000)
    plant(buf, 9000, 9000 - 777, 9)
    plant(buf, 9021, 9021 - 777, 9)
    out.append(Case("rep", "repeat-along-one-path", [buf]))
    buf = rand(rng, 30000)
    plant(buf, 8000, 9000, 12)                  # offsets 1000 and 1012 cost the same (code 9): the smaller is kept
    plant(buf, 7988, 9000, 12)
    out.append(Case("rep", "cost-tie-smaller-offset", [buf]))
    return out


def segment_ends(rng):
    """A 64-byte repeat straddling segment starts: no match crosses its segment's end."""
    buf = rand(rng, BLOCK)
    for w in range(1, CM_WARPS):
        s = seg_bounds(BLOCK, w)[0]
        plant(buf, s - 32, s - 5000, 64)
    return [Case("segend", "straddle-every-segment-start", [buf])]


def chains(rng):
    """Sources at the chain's reach: offsets 131072 and 131073 into the previous block, and at the frame's start."""
    out = []
    for d in (WINDOW, WINDOW + 1):
        buf = rand(rng, 2 * BLOCK)
        plant(buf, BLOCK + 5000, BLOCK + 5000 - d, 24)
        out.append(Case("chain", f"offset-{d}" + ("=WINDOW" if d == WINDOW else "=WINDOW+1"), [buf]))
    buf = rand(rng, 3000)
    plant(buf, 2000, 0, 30)
    out.append(Case("chain", "source-at-frame-start", [buf]))
    return out


def realistic():
    return [Case("data", c.id.split("-", 1)[1], c.frames, c.content) for c in cparse.cases("data")]


GROUPS = {"suff": suff, "wincap": window_cap, "rep": repeats, "segend": segment_ends, "chain": chains}
SHAPES = ("n1=one", "n5=MIN_MATCH", "n41=41", "n131072=BLOCK", "n131073=BLOCK+1", "n131078=BLOCK+6")


def cases(group=None):
    """The crafted cases (all groups, or one), built from fixed seeds, plus some of the Fastest model's shapes, its RLE, dense,
    isolation and dictionary cases, LAZY's repeat cases and the realistic group."""
    out = []
    for i, (g, fn) in enumerate(GROUPS.items()):
        if group is None or g == group:
            out += fn(random.Random(0x0B7 + i))
    if group is None or group == "shape":
        out += [Case("shape", c.id.split("-", 1)[1], c.frames, c.content) for c in cparse.cases("shape") if c.id.split("-", 1)[1] in SHAPES]
    for g in ("rle", "dense", "isolation", "dict"):
        if group is None or group == g:
            out += [Case(g, c.id.split("-", 1)[1], c.frames, c.content) for c in cparse.cases(g)]
    if group is None or group == "lazyrep":
        out += [Case("lazyrep", c.id.split("-", 1)[1], c.frames, c.content) for c in clazy.cases("rep")]
    if group is None or group == "data":
        out += realistic()
    return out
