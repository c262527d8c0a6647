"""The compressor's parse written out plainly: what k_cmatch must produce for every block, and the frame the compressor must write.

This module restates the rules of zstd-rs_b200/csrc/compress.cu (k_cmatch) and DESIGN.md section 4.4 in Python, calling nothing in
the library.  `parse` gives, for every 128 KiB block of every frame of a submission, either ("rle", byte, n) or (literals,
[(ll, ml, of), ...]) -- exactly what k_cmatch packs, `of` being the actual offset (the encoder codes it as of + 3).  An empty block
(the empty frame's only one) is (b"", []).  The rules:

  blocks    frames are cut into 128 KiB blocks; a block's `back` is min(its position in the frame, 131072).  A non-empty block
            whose bytes are all equal is RLE.
  hash      hash5(p, log) = ((le40(p) << 24) * 889523592379 mod 2^64) >> (64 - log); log 14 (t1), 12 (tp), 17 (dictionary).
  t1        per hash, the smallest q of the block with q + 5 <= n.
  segments  8 per block: seglen = ceil(n / 8), s = min(n, w * seglen), e = min(n, s + seglen); some may be empty.
  tp        per segment, the most recent position per hash, seeded with every q in [max(s - 16384, -min(back, 16384)), s) with
            q + 5 <= n (the seeds may lie in the previous block of the same frame, never in another frame).
  rounds    32 positions at a time from p: every lane q in [p, p + 32) with q + 5 <= e looks up t1 and tp as they stood before
            the round, then every such lane inserts q into tp (lanes past the chosen match too).  The t1 candidate counts when
            c1 < q, the tp candidate when c2 < q and q - c2 <= 131072.  Each is verified for up to min(16, e - q) bytes; the longer
            wins, the smaller offset on equal length.  The first lane with a match of >= 5 bytes is taken; a match of exactly 16
            bytes is extended up to e.  The next round starts at qj + ml; a round without a match advances p by 32.
            A tp offset is below 32 KiB by construction (c2 >= s - 16384 and q < s + 16384), so its window check never fails;
            offsets up to 131071 come from t1 only.
  dictionary  only the content's last min(len, 131072) bytes count; its table holds, per hash, the most recent d with
            d + 5 <= len.  A lane looks it up when len >= 5 and back + q < 131072; the candidate's offset back + q + len - d must
            be <= 131072; it is verified for min(16, e - q, len - d) bytes and extended only up to the dictionary's end; it
            replaces the in-frame candidate when longer, or as long with a smaller offset.
  packing   a segment's trailing literals join the next segment's first sequence, across any segments without sequences; the
            last segments' literals are the block's trailing literals.
  header    Single_Segment 0; Window_Descriptor exponent min(window_log, max(17, ceil(log2 n))), mantissa 0.

The block and frame drivers are shared by every level: a `Level` names its hash logs, its segment loop (`_segment` here, LAZY's in
tests/clazy.py) and the records its blocks are coded from.  A segment loop also takes the segment's forced pieces, the long matches
of tests/cldm.py clipped to it (none at window_log 17).  `reference_frame` assembles the frame from the parse (header, blocks
through tests/cenc.py's plain statement of the entropy stage, checksum), and `xxh64` is XXH64 with seed 0.  `cases()` builds the crafted inputs the tests run; each case's id names the constant it sits on."""
import bisect
import collections
import random
import struct

import numpy as np

import cenc

BLOCK = 131072          # ENC_BLOCK
WINDOW = 131072         # ENC_WINDOW
WINDOW_LOG_MIN = 17     # B200Z_WINDOW_LOG_MIN (2^17 = WINDOW)
MIN_MATCH = 5           # ENC_MIN_MATCH
CM_WARPS = 8            # segments per block
CM_T1_LOG, CM_TP_LOG, CD_LOG = 14, 12, 17
CM_SEED = 16384         # bytes before its segment a segment's tp is seeded from
CM_CAP = 16             # bytes a lane verifies before the chosen match is extended
CSEG_SEQS = (BLOCK // CM_WARPS) // MIN_MATCH + 1   # sequences one segment can hold (3277)
HASH_MUL = 889523592379

# statistics bins of the dictionary finalizer (DS_* in csrc/compress.h)
DS_LIT, DS_LL, DS_ML, DS_OF = 0, 256, 256 + 36, 256 + 36 + 53
DS_BINS = DS_OF + 32
DS_BLOCKS = 2048
# code baselines of RFC 8878 section 3.1.1.3.2.1.1: a value's code is the last one whose baseline does not exceed it
LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64] + [1 << k for k in range(7, 17)]
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99] + [(1 << k) + 3 for k in range(7, 17)]


def hashes(buf, log):
    """hash5 of every position p of buf with p + 5 <= len(buf), as a list."""
    a = np.frombuffer(bytes(buf), dtype=np.uint8).astype(np.uint64)
    n = len(a) - 4
    if n <= 0:
        return []
    v = a[:n] | (a[1:n + 1] << np.uint64(8)) | (a[2:n + 2] << np.uint64(16)) | (a[3:n + 3] << np.uint64(24)) | (a[4:n + 4] << np.uint64(32))
    with np.errstate(over="ignore"):
        h = ((v << np.uint64(24)) * np.uint64(HASH_MUL)) >> np.uint64(64 - log)
    return h.tolist()


class Dictionary:
    """The part of a dictionary's content a match can reach (its last min(len, 131072) bytes) and its match table."""

    def __init__(self, content):
        self.data = bytes(content)[-WINDOW:] if content else b""
        self.n = len(self.data)
        self.tab = {}
        for d, h in enumerate(hashes(self.data, CD_LOG)):
            self.tab[h] = d                     # the most recent position wins


def _mlen(a, i, b, j, lim):
    n = 0
    while n < lim and a[i + n] == b[j + n]:
        n += 1
    return n


def _segment(F, base, n, back, s, e, t1, H14, H12, H17, dic, pieces):
    """Parse of segment [s, e) of the block at F[base:base + n] with its forced pieces [(cs, ce, off)] (empty: none): (literals,
    sequences, trailing literal count)."""
    tp = {}
    for q in range(max(s - CM_SEED, -min(back, CM_SEED)), min(s, n - MIN_MATCH + 1)):
        tp[H12[base + q]] = q
    seqs, lits = [], []
    p = anchor = s
    for k in range(len(pieces) + 1):
        stop = pieces[k][0] if k < len(pieces) else e   # the parse runs up to the next piece's start
        last = stop - MIN_MATCH + 1             # lanes q < last have q + 5 <= stop
        while p < last:
            hi = min(p + 32, last)
            found = None
            for q in range(p, hi):
                fq = base + q
                lim = min(CM_CAP, stop - q)
                best = cand = 0
                c1 = t1[H14[fq]]
                if c1 < q:
                    best, cand = _mlen(F, fq, F, base + c1, lim), q - c1
                c2 = tp.get(H12[fq])
                if c2 is not None and c2 < q and q - c2 <= WINDOW:
                    l2 = _mlen(F, fq, F, base + c2, lim)
                    if l2 > best or (l2 == best and q - c2 < cand):
                        best, cand = l2, q - c2
                xlim = stop - q
                if dic is not None and back + q < WINDOW:
                    d = dic.tab.get(H17[fq])
                    if d is not None and back + q + dic.n - d <= WINDOW:
                        off3, rest = back + q + dic.n - d, dic.n - d
                        l3 = _mlen(F, fq, dic.data, d, min(lim, rest))
                        if l3 > best or (l3 == best and off3 < cand):
                            best, cand, xlim = l3, off3, min(xlim, rest)
                if best >= MIN_MATCH:
                    found = (q, best, cand, xlim)
                    break
            for q in range(p, hi):              # every valid lane inserts, before or after the chosen one
                h = H12[base + q]
                if tp.get(h, -WINDOW - 1) < q:
                    tp[h] = q
            if found is None:
                p += 32
                continue
            q, ml, off, xlim = found
            if ml == CM_CAP:
                fq = base + q
                if off > back + q:              # the source lies in the dictionary: stop at its end
                    ref, r0 = dic.data, dic.n - (off - (back + q))
                else:
                    ref, r0 = F, fq - off
                while ml < xlim and F[fq + ml] == ref[r0 + ml]:
                    ml += 1
            lits.append(F[base + anchor:base + q])
            seqs.append((q - anchor, ml, off))
            anchor = p = q + ml
        if k < len(pieces):                     # the piece is one sequence; the parse resumes at its end
            cs, ce, off = pieces[k]
            lits.append(F[base + anchor:base + cs])
            seqs.append((cs - anchor, ce - cs, off))
            anchor = p = ce
    lits.append(F[base + anchor:base + e])
    assert len(seqs) <= CSEG_SEQS
    return b"".join(lits), seqs, e - anchor


def raw_offsets(seqs):
    """Fastest's records: every offset is coded raw (Offset_Value = of + 3), so the encoder takes the sequences as parsed."""
    return seqs


# A level's parse: the hash logs of its t1 and of its segments' tables, its segment loop, and the records its blocks are coded
# from (reference_frame).  UNCOMPRESSED has no parse: every block is Raw.
Level = collections.namedtuple("Level", "t1_log tab_log segment records")
FASTEST = Level(CM_T1_LOG, CM_TP_LOG, _segment, raw_offsets)
UNCOMPRESSED = None


def _pieces(kept, s, e):
    """A block's kept long matches [(start, length, offset)] clipped to segment [s, e): [(cs, ce, off)], pieces under MIN_MATCH
    bytes dropped."""
    out = []
    for st, ln, off in kept:
        if st >= e:
            break
        cs, ce = max(st, s), min(st + ln, e)
        if ce >= cs + MIN_MATCH:
            out.append((cs, ce, off))
    return out


def parse_block(F, base, n, back, level, H_t1, H_tab, H17, dic, kept=()):
    """One block of frame F: ("rle", byte, n), or (literals, [(ll, ml, of), ...]); (b"", []) for the empty block.  kept: the
    block's long matches (tests/cldm.py), taken as forced pieces."""
    blk = F[base:base + n]
    if n == 0:
        return (b"", [])
    if blk.count(blk[:1]) == n:
        return ("rle", blk[0], n)
    t1 = [BLOCK] * (1 << level.t1_log)
    for q in range(n - MIN_MATCH, -1, -1):      # the smallest position wins
        t1[H_t1[base + q]] = q
    seglen = -(-n // CM_WARPS)
    lits, seqs, carry = [], [], 0
    for w in range(CM_WARPS):
        s = min(n, w * seglen)
        e = min(n, s + seglen)
        sl, ss, trail = level.segment(F, base, n, back, s, e, t1, H_t1, H_tab, H17, dic, _pieces(kept, s, e))
        lits.append(sl)
        if ss:
            ss[0] = (ss[0][0] + carry, ss[0][1], ss[0][2])
            carry = trail
        else:
            carry += trail
        seqs += ss
    return (b"".join(lits), seqs)


def parse_frame(data, level=FASTEST, dic=None, kept=None):
    """The blocks of one frame at `level` (see parse_block); dic: a Dictionary or None; kept: the frame's long matches, one list
    per block (cldm.forced), or None."""
    F = bytes(data)
    H_t1, H_tab = hashes(F, level.t1_log), hashes(F, level.tab_log)
    H17 = hashes(F[:WINDOW + 4], CD_LOG) if dic is not None else None
    out, pos = [], 0
    while True:
        n = min(BLOCK, len(F) - pos)
        out.append(parse_block(F, pos, n, min(pos, WINDOW), level, H_t1, H_tab, H17, dic, kept[len(out)] if kept else ()))
        pos += n
        if pos >= len(F):
            return out


def match_dict(content):
    """The Dictionary a raw-content or formatted dictionary's content gives k_cmatch, or None when it has < 5 bytes."""
    return Dictionary(content) if content is not None and len(content) >= MIN_MATCH else None


def parse(frames, content=None, level=FASTEST, kept=None):
    """The parse of every frame of one submission at `level`, against a dictionary's content (raw content or a formatted
    dictionary's); kept: per frame, its long matches per block (cldm.forced), or None."""
    dic = match_dict(content)
    return [parse_frame(f, level, dic, kept[i] if kept else None) for i, f in enumerate(frames)]


# ---------------------------------------------------------------------------------------------------------------------------
# XXH64 and the reference frame
# ---------------------------------------------------------------------------------------------------------------------------
_M = (1 << 64) - 1
P1, P2, P3, P4, P5 = 0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63, 0x27D4EB2F165667C5


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & _M


def _round(acc, v):
    return (_rotl((acc + v * P2) & _M, 31) * P1) & _M


def xxh64(data):
    """XXH64 of data, seed 0 (the xxHash specification)."""
    b = bytes(data)
    n, p = len(b), 0
    if n >= 32:
        v = [(P1 + P2) & _M, P2, 0, (-P1) & _M]
        words = struct.unpack_from(f"<{(n // 32) * 4}Q", b)
        for i in range(0, len(words), 4):
            v = [_round(v[0], words[i]), _round(v[1], words[i + 1]), _round(v[2], words[i + 2]), _round(v[3], words[i + 3])]
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M
        for x in v:
            h = ((h ^ _round(0, x)) * P1 + P4) & _M
        p = (n // 32) * 32
    else:
        h = P5
    h = (h + n) & _M
    while p + 8 <= n:
        h = (_rotl(h ^ _round(0, struct.unpack_from("<Q", b, p)[0]), 27) * P1 + P4) & _M
        p += 8
    if p + 4 <= n:
        h = (_rotl(h ^ ((struct.unpack_from("<I", b, p)[0] * P1) & _M), 23) * P2 + P3) & _M
        p += 4
    while p < n:
        h = (_rotl(h ^ ((b[p] * P5) & _M), 11) * P1) & _M
        p += 1
    h = ((h ^ (h >> 33)) * P2) & _M
    h = ((h ^ (h >> 29)) * P3) & _M
    return h ^ (h >> 32)


_tables = {}


def encode_with_tables(formatted, lits, seqs):
    """Content of a frame's first Compressed block coded with a formatted dictionary's tables (tests/cenc.py)."""
    key = bytes(formatted)
    if key not in _tables:
        _tables[key] = cenc.Tables(key)
    return cenc.encode_block(lits, seqs, _tables[key])[0]


def dict_id_field(dict_id):
    return 0 if dict_id == 0 else 1 if dict_id < 256 else 2 if dict_id < 65536 else 4


def frame_window_log(n, window_log):
    """The Window_Descriptor exponent of a frame of n bytes compressed at window_log: min(window_log, max(17, ceil(log2 n)))."""
    if window_log <= WINDOW_LOG_MIN:
        return WINDOW_LOG_MIN
    c = WINDOW_LOG_MIN
    while c < window_log and (1 << c) < n:
        c += 1
    return c


def frame_header(n, checksum, dict_id=0, window_log=WINDOW_LOG_MIN):
    """Single_Segment 0, the window of frame_window_log (mantissa 0), the dictionary ID in its smallest field, Frame_Content_Size
    in its smallest legal one."""
    did = dict_id_field(dict_id)
    fcs = struct.pack("<H", n - 256) if 256 <= n <= 65791 else struct.pack("<Q", n) if n >> 32 else struct.pack("<I", n)
    flag = {2: 1, 4: 2, 8: 3}[len(fcs)]
    fhd = (flag << 6) | (4 if checksum else 0) | {0: 0, 1: 1, 2: 2, 4: 3}[did]
    wd = (frame_window_log(n, window_log) - 10) << 3
    return struct.pack("<IBB", 0xFD2FB528, fhd, wd) + dict_id.to_bytes(did, "little") + fcs


def reference_frame(data, blocks, checksum=True, dict_id=0, dict_tables=None, level=FASTEST, window_log=WINDOW_LOG_MIN):
    """The frame the compressor must write for `data` whose parse at `level` is `blocks` (parse_frame) at window_log.  At
    UNCOMPRESSED every block is Raw.  dict_tables: the formatted dictionary whose tables code the frame's first block
    (compress_frames(..., dict_tables=True))."""
    data = bytes(data)
    out = frame_header(len(data), checksum, dict_id, window_log)
    pos = 0
    for k, b in enumerate(blocks):
        last = 1 if k + 1 == len(blocks) else 0
        n = min(BLOCK, len(data) - pos)
        raw = data[pos:pos + n]
        if level is not UNCOMPRESSED and b[0] == "rle":
            out += struct.pack("<I", last | (1 << 1) | (n << 3))[:3] + bytes([b[1]])
        else:
            content = None
            if level is not UNCOMPRESSED and n:
                recs = level.records(b[1])
                if dict_tables is not None and k == 0:
                    content = encode_with_tables(dict_tables, b[0], recs)
                else:
                    content = cenc.encode_block(b[0], recs)[0]
            if content is not None and len(content) < n:
                out += struct.pack("<I", last | (2 << 1) | (len(content) << 3))[:3] + content
            else:
                out += struct.pack("<I", last | (n << 3))[:3] + raw
        pos += n
    if checksum:
        out += struct.pack("<I", xxh64(data) & 0xFFFFFFFF)
    return out


def ll_code(v):
    return bisect.bisect_right(LL_BASE, v) - 1


def ml_code(v):
    return bisect.bisect_right(ML_BASE, v) - 1


def counts(samples, content):
    """The dictionary finalizer's statistics: each sample's first 131072 bytes parsed as a frame's first block against the content,
    RLE samples left out; literal bytes, LL / ML codes and OF codes (of offset + 3), as in k_dstats."""
    dic = match_dict(content)
    cnt = np.zeros(DS_BINS, dtype=np.uint64)
    for smp in samples:
        b = parse_frame(bytes(smp)[:BLOCK], FASTEST, dic)[0]
        if b[0] == "rle":
            continue
        lits, seqs = b
        cnt[DS_LIT:DS_LIT + 256] += np.bincount(np.frombuffer(lits, dtype=np.uint8), minlength=256).astype(np.uint64)
        for ll, ml, of in seqs:
            cnt[DS_LL + ll_code(ll)] += 1
            cnt[DS_ML + ml_code(ml)] += 1
            cnt[DS_OF + (of + 3).bit_length() - 1] += 1
    return cnt


# ---------------------------------------------------------------------------------------------------------------------------
# the crafted cases
# ---------------------------------------------------------------------------------------------------------------------------
class Case:
    """One submission's worth of frames (usually one) and the dictionary content they are compressed against (None: none)."""

    def __init__(self, group, name, frames, content=None):
        self.group, self.id = group, f"{group}-{name}"
        self.frames = [bytes(f) for f in frames]
        self.content = None if content is None else bytes(content)

    def __repr__(self):
        return self.id


def rand(rng, n):
    return bytearray(rng.getrandbits(8) for _ in range(n))


def plant(buf, dst, src, n, ref=None):
    """Copies n bytes from src (of ref, default buf) to dst and makes the bytes around the copy differ from the source's
    neighbours, so that the repeat is exactly n bytes long."""
    ref = buf if ref is None else ref
    n = min(n, len(buf) - dst)
    buf[dst:dst + n] = ref[src:src + n]
    if dst + n < len(buf) and src + n < len(ref) and buf[dst + n] == ref[src + n]:
        buf[dst + n] ^= 0x5A
    if dst > 0 and src > 0 and buf[dst - 1] == ref[src - 1]:
        buf[dst - 1] ^= 0xA5


def seg_bounds(n, w):
    seglen = -(-n // CM_WARPS)
    s = min(n, w * seglen)
    return s, min(n, s + seglen)


def _sprinkle(rng, buf, lo, hi, every=3000, reach=8000):
    """Repeats of 6-40 bytes every `every` bytes in [lo, hi), sources up to `reach` bytes back inside [lo, hi)."""
    for dst in range(lo + reach // 2, hi - 64, every):
        n = rng.randint(6, 40)
        src = rng.randint(max(lo, dst - reach), dst - n - 1)
        plant(buf, dst, src, n)


def shapes(rng):
    out = []
    names = {1: "one", 4: "MIN_MATCH-1", 5: "MIN_MATCH", 6: "MIN_MATCH+1", 7: "7", 8: "CM_WARPS", 9: "CM_WARPS+1", 41: "41",
             CM_SEED * 8 - 1: "8*CM_SEED-1", CM_SEED * 8 + 1: "8*CM_SEED+1", BLOCK - 1: "BLOCK-1", BLOCK: "BLOCK", BLOCK + 1: "BLOCK+1"}
    for k in range(2, 7):
        names[BLOCK + k] = f"BLOCK+{k}"
    for n, name in names.items():
        buf = rand(rng, n)
        if n == 41:
            plant(buf, 30, 2, 9)
        _sprinkle(rng, buf, 0, n)
        if n > BLOCK:                           # the last block repeats the first block's tail
            plant(buf, BLOCK, BLOCK - 300, n - BLOCK)
        out.append(Case("shape", f"n{n}={name}", [buf]))
    # segments without a sequence carry their bytes on: m quiet segments at the start, in the middle and at the end
    for m in range(1, 8):
        for where in ("head", "mid", "tail"):
            if where == "mid" and m > 6:
                continue
            first = {"head": 0, "mid": 1, "tail": CM_WARPS - m}[where]
            quiet = set(range(first, first + m))
            buf = rand(rng, BLOCK)
            for w in range(CM_WARPS):
                if w not in quiet:
                    s, e = seg_bounds(BLOCK, w)
                    _sprinkle(rng, buf, s, e, every=2500, reach=4000)
            out.append(Case("carry", f"{m}-quiet-segments-{where}", [buf]))
    return out


def segment_ends(rng):
    """A 64-byte repeat straddling each of the 8 segment starts (segment 0's is the second block's first byte)."""
    out = []
    for w in range(CM_WARPS):
        buf = rand(rng, 2 * BLOCK)
        s = BLOCK + seg_bounds(BLOCK, w)[0]
        plant(buf, s - 32, s - 5000, 64)
        out.append(Case("segend", f"straddle-segment{w}-start", [buf]))
    return out


def rounds(rng):
    out = []
    s1 = seg_bounds(20000, 1)[0]                # segment 1 runs in rounds of 32 from s1 until its first match
    for lane in (0, 31):
        buf = rand(rng, 20000)
        plant(buf, s1 + 320 + lane, 500, 20)
        out.append(Case("round", f"match-at-lane{lane}", [buf]))
    buf = rand(rng, 20000)
    plant(buf, s1 + 320 + 3, 400, 8)            # taken; the round's second match is found again from qj + ml
    plant(buf, s1 + 320 + 20, 900, 10)
    out.append(Case("round", "two-matches-one-round", [buf]))
    buf = rand(rng, BLOCK)
    for w in range(CM_WARPS):
        s, e = seg_bounds(BLOCK, w)
        plant(buf, e - MIN_MATCH, s + 10 + w, MIN_MATCH)   # the segment's last valid lane, q + 5 == e
    out.append(Case("round", "match-at-q+5=e", [buf]))
    return out


def cap(rng):
    out = []
    for n in (5, 15, 16, 17, 47, 48, 49):
        buf = rand(rng, 30000)
        plant(buf, 7000, 1234, n)
        plant(buf, 20000 + n, 19000, n)         # and once more, its source earlier in the same segment
        out.append(Case("cap", f"ml{n}" + ("=CM_CAP" if n == CM_CAP else f"=CM_CAP{n - CM_CAP:+d}" if abs(n - CM_CAP) == 1 else ""), [buf]))
    # in every segment a 40-byte repeat from 300 bytes before e, its source kept in tp until the lane at its copy looks it up
    buf = rand(rng, BLOCK)
    for w in range(CM_WARPS):
        s, e = seg_bounds(BLOCK, w)
        plant(buf, e - 40, e - 300, 40)         # a match longer than CM_CAP that runs exactly to e
        keep_in_tp(buf, e - 300, e - 40, set(range(e - 301, e - 259)) | set(range(e - 41, e)))
    out.append(Case("cap", "extension-to-e", [buf]))
    buf = rand(rng, BLOCK)
    for w in range(CM_WARPS):
        s, e = seg_bounds(BLOCK, w)
        plant(buf, e - 16, e - 300, 40)         # e - q == CM_CAP: no extension possible; the next segment takes the rest
        protect = set(range(e - 301, e - 259)) | set(range(e - 17, e + 24))
        keep_in_tp(buf, e - 300, e - 16, protect)
        keep_in_tp(buf, e - 284, e, protect)
    out.append(Case("cap", "e-q=CM_CAP", [buf]))
    return out


def hash5(buf, p, log):
    return (((int.from_bytes(bytes(buf[p:p + 5]), "little") << 24) * HASH_MUL) & _M) >> (64 - log)


def keep_in_tp(buf, first, dst, protect):
    """Changes bytes of buf so that no position in (first, dst) shares position first's tp hash: the entry of `first` is then
    still tp's when the lane at dst looks it up.  Bytes in `protect` are left alone."""
    target = hash5(buf, first, CM_TP_LOG)
    while True:
        bad = [p for p in range(first + 1, dst) if hash5(buf, p, CM_TP_LOG) == target]
        if not bad:
            return
        for p in bad:
            i = next(i for i in range(p, p + 5) if i not in protect)
            buf[i] ^= 0x3C


def seeds(rng):
    """A source exactly CM_SEED bytes before a segment start (the oldest seed of its tp) and one CM_SEED + 1 before (not seeded;
    its second position is), in the last block of a 2- and a 3-block frame, where t1 cannot see it; no later position shares
    the seed's tp hash.  The same distances inside one block, where t1 may still find the source."""
    out = []
    for nblocks in (2, 3):
        for d in (CM_SEED, CM_SEED + 1):
            buf = rand(rng, nblocks * BLOCK)
            b = (nblocks - 1) * BLOCK           # the last block: segment 0 starts at its first byte
            plant(buf, b + 2000, b - d, 24)
            keep_in_tp(buf, b - CM_SEED, b + 2000, set(range(b - d - 1, b - d + 25)) | set(range(b + 1999, b + 2025)))
            s1 = b + seg_bounds(BLOCK, 3)[0]    # segment 3: the source lies in the same block (t1 may find it)
            plant(buf, s1 + 700, s1 - d, 24)
            out.append(Case("seed", f"{nblocks}blocks-source-{d}-before-segment" + ("=CM_SEED" if d == CM_SEED else "=CM_SEED+1"), [buf]))
    return out


def choice(rng):
    """A string three times in a block: at x (t1's candidate), y (tp's) and z; the first two match z for a chosen length."""
    out = []
    for name, (lx, ly) in {"t1-longer": (12, 9), "tp-longer": (9, 12), "equal-smaller-offset": (11, 11)}.items():
        buf = rand(rng, 40000)
        x, y, z = 1000, 8000, 9000              # x in segment 0, y and z in segment 1 (seglen 5000): y is in z's tp
        plant(buf, z, 20000, 20)
        plant(buf, x, z, lx)
        plant(buf, y, z, ly)
        out.append(Case("choice", name, [buf]))
    return out


def isolation(rng):
    a = rand(rng, 5000)
    b = a[-200:] + rand(rng, 3000)
    big = rand(rng, BLOCK + 7000)
    c = big[-300:] + rand(rng, 2000)
    return [Case("isolation", "second-frame-starts-with-first-tail", [a, b]),
            Case("isolation", "after-two-block-frame", [big, c])]


def dense(rng):
    """5-byte chunks copied from a random prefix: about seglen / 5 sequences per segment, close to CSEG_SEQS."""
    pre = 2048
    buf = rand(rng, BLOCK)
    for dst in range(pre, BLOCK - 5, 5):
        src = rng.randrange(0, pre - 6)
        buf[dst:dst + 5] = buf[src:src + 5]
    return [Case("dense", f"5-byte-chunks-CSEG_SEQS={CSEG_SEQS}", [buf])]


def rle(rng):
    a, c = rand(rng, BLOCK), rand(rng, 5000)
    mid = b"\x61" * BLOCK
    nearly = bytearray(b"\x00" * BLOCK)
    nearly[-1] = 1
    return [Case("rle", "rle-block-between-two", [a + mid + c]),
            Case("rle", "equal-but-last-byte", [nearly]),
            Case("rle", "empty-frame", [b""])]


def dictionaries(rng):
    out = []
    for k in (4, 5, 6):
        content = rand(rng, k)
        f = bytearray(content) + rand(rng, 300) + content + rand(rng, 20)
        out.append(Case("dict", f"len{k}" + ("=MIN_MATCH" if k == MIN_MATCH else f"=MIN_MATCH{k - MIN_MATCH:+d}"), [f], content))
    big = rand(rng, 200000)
    f = rand(rng, 20000)
    plant(f, 3000, 1000, 30, big)               # only in the head: beyond the 128 KiB tail, unreachable
    plant(f, 9000, len(big) - 5000, 30, big)
    out.append(Case("dict", "longer-than-WINDOW-head-and-tail", [f], big))
    content = rand(rng, WINDOW)
    f = rand(rng, 6000)
    plant(f, 1000, 1000, 20, content)           # offset back + q + len - d = WINDOW
    plant(f, 2000, 1999, 20, content)           # WINDOW + 1: refused
    out.append(Case("dict", "offset=WINDOW-and-WINDOW+1", [f], content))
    content = rand(rng, 3000)
    f = rand(rng, 4000)
    for i, left in enumerate((16, 17, 40)):      # a match ending exactly at the dictionary's end
        f[500 + 1000 * i:500 + 1000 * i + left] = content[-left:]
        # then the dictionary's first 30 bytes: a second dictionary match must start exactly where the first stops.  The GPU
        # is held to that split; whether an extension stays inside the dictionary is checked in the model only (an overrun
        # there would index past the tail), since the bytes after the dictionary's tail on the device are not the input's
        f[500 + 1000 * i + left:500 + 1000 * i + left + 30] = content[:30]
    out.append(Case("dict", "ends-at-dict-end-16-17-40", [f], content))
    content = rand(rng, 3000)
    f = rand(rng, 30000)
    plant(f, 100, 2000, 40, content)
    plant(f, 20000, 2000, 40, content)          # in-frame source (offset 19900) as long as the dictionary's
    out.append(Case("dict", "in-frame-as-long-as-dict", [f], content))
    content = rand(rng, 3000)
    plant(content, 2500, 600, 24)               # the later occurrence wins
    f = rand(rng, 2000)
    plant(f, 700, 600, 24, content)
    out.append(Case("dict", "twice-in-dict-later-wins", [f], content))
    content = rand(rng, 3000)
    f = rand(rng, BLOCK + 5000)
    plant(f, BLOCK + 1000, 500, 30, content)    # second block: no dictionary lookup
    plant(f, 50000, 700, 30, content)
    out.append(Case("dict", "no-lookup-in-second-block", [f], content))
    return out


def realistic():
    import datagen
    out = [Case("data", "gen_text-3-blocks", [datagen.gen_text(3 * BLOCK + 777, 0xC9A1)]),
           Case("data", "gen_silesia_mix-2-blocks", [datagen.gen_silesia_mix(2 * BLOCK, 0xC9A2)]),
           Case("data", "gen_binary_records-2-blocks", [datagen.gen_binary_records(2 * BLOCK - 3, 0xC9A3)])]
    fs = datagen.config_c5(nframes=200, cache=False)
    plain = fs.plain.tobytes()
    pieces = [plain[int(o):int(o + n)] for o, n in zip(fs.out_off, fs.out_size)]
    out.append(Case("data", "c5-200-pieces-raw-content", pieces, fs.raw_dict.tobytes()))
    return out


GROUPS = {"shape": shapes, "segend": segment_ends, "round": rounds, "cap": cap, "seed": seeds, "choice": choice,
          "isolation": isolation, "dense": dense, "rle": rle, "dict": dictionaries}


def cases(group=None):
    """The crafted cases (all groups, or one), built from fixed seeds; "data" is the realistic group."""
    out = []
    for i, (g, fn) in enumerate(GROUPS.items()):
        if group is None or g == group:
            out += fn(random.Random(0xC0A5 + i))
    if group is None or group == "data":
        out += realistic()
    return out
