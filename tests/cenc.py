"""The compressor's entropy stage written out plainly: the bytes k_cenc (encode_block of zstd-rs_b200/csrc/encode.cuh) writes for a
block's literals and sequences, and the dictionary writer's header (dict_format.cpp).

Nothing here runs encode.cuh.  The format's writers are tests/entcraft.py's (write_ncount, fse_table, huf_weights, huf_table,
write_huf_desc, huf_stream, seq_bitstream, lit_header); this module states only the encoder's decisions, in the order encode.cuh
makes them.  Records are (ll, ml, of) with of = Offset_Value - 3 mod 2^32, as k_cenc hands them to encode_block (Fastest's raw
offsets, or a level's repeat records).

  literals   byte histogram.  Raw when n <= 1024, when there is one distinct byte, when the Huffman description cannot be
             written, or when hsize + csize >= n + 3; else own Huffman in 4 streams of (n + 3) / 4.  hsize is 4 when both n
             and csize are below 16384, else 5; csize = description + 6 + the streams.  Raw headers take 1, 2 or 3 bytes.
  huf_lengths  stable sort by (count, symbol); a two-queue merge that takes the leaf on a tie; depths clamped to 11; while the
             Kraft sum is above 1, lengthen the longest code that can still grow, rarest first; while below, shorten the longest
             code, most frequent first.  Codes are canonical in the decoder's order (huf_table).
  weights    direct 4-bit form when there are at most 128 of them; else FSE-compressed at accuracy log 6 with two interleaved
             states; no description when that body takes 128 bytes or more or when only one weight value occurs.
  sequences  the count in 1, 2 or 3 bytes; per LL / OF / ML table RLE for a single code, else FSE_Compressed at fse_pick_log with
             fse_normalize's counts; the bitstream is seq_bitstream's (OF, ML, LL state updates, ML, OF, LL flush) with every
             chain ending in its code's first state (FSE_initCState's choice for this spread).
  dictionary (a formatted dictionary's tables, a frame's first block only) Treeless literals -- 1 stream below 1024 literals,
             else 4 -- when every literal byte has a code and the result is strictly smaller than the choice above (a 1-stream
             result of 1024 bytes or more is refused); Repeat per table when it has more than one code, each present in the
             dictionary's table, and fse_cost_q8(dictionary) <= description * 2^11 + fse_cost_q8(own).
  block      RLE when all bytes are equal, Compressed when the content is smaller than the block, else Raw (k_cenc, k_cassemble).
"""
import struct

import numpy as np

import entcraft as E

HUF_MAX_BITS = 11               # ENC_HUF_MAX_BITS
RAW_LITERALS_MAX = 1024         # ENC_RAW_LITERALS_MAX
WEIGHTS_DIRECT_MAX = 128        # weights the direct 4-bit form can hold
WEIGHTS_LOG = 6                 # accuracy log of FSE-compressed weights
LIT_HEADER_4_MAX = 16384        # n and csize below it: the 4-byte compressed-literals header
TREELESS_1_STREAM = 1024        # Treeless literals below it: one stream
MAX_LOG = (9, 8, 9)             # LL, OF, ML accuracy logs (compressed.rs:55-72)
MAX_SYM = (35, 31, 52)
LL, OF, ML = 0, 1, 2
RAW, HUF, TREELESS = 0, 1, 3    # literal modes as the host drivers print them
RLE_MODE, FSE_MODE, REPEAT_MODE = 1, 2, 3
LL_BASE = np.array(E.LL_BASE)
ML_BASE = np.array(E.ML_BASE)


# ---------------------------------------------------------------------------------------------------------------------------
# Huffman
# ---------------------------------------------------------------------------------------------------------------------------
def huf_lengths(cnt, steps=None):
    """Code lengths {symbol: length} for counts cnt[256] (>= 2 nonzero): limited to 11 and Kraft-complete.  steps: a list that
    gets ("grow", symbol) / ("shrink", symbol) for every fix-up step."""
    order = sorted((int(c), s) for s, c in enumerate(cnt) if c)        # stable by (count, symbol)
    n = len(order)
    w = [c for c, _ in order]
    parent = [0] * (2 * n - 1)
    a, b = 0, n                                 # leaves [a, n), internal nodes [b, len(w))
    for k in range(n, 2 * n - 1):
        pick = []
        for _ in range(2):
            if a < n and (b >= k or w[a] <= w[b]):
                pick.append(a)
                a += 1
            else:
                pick.append(b)
                b += 1
        w.append(w[pick[0]] + w[pick[1]])
        parent[pick[0]] = parent[pick[1]] = k
    depth = [0] * (2 * n - 1)
    for k in range(2 * n - 3, -1, -1):
        depth[k] = depth[parent[k]] + 1
    ln = [min(depth[i], HUF_MAX_BITS) for i in range(n)]        # by rank, rarest first
    one = 1 << HUF_MAX_BITS
    kraft = sum(1 << (HUF_MAX_BITS - x) for x in ln)
    while kraft > one:                          # lengthen the longest code that can still grow, rarest first
        m = max((i for i in range(n) if ln[i] < HUF_MAX_BITS), key=lambda i: (ln[i], -i))
        ln[m] += 1
        kraft -= 1 << (HUF_MAX_BITS - ln[m])
        if steps is not None:
            steps.append(("grow", order[m][1]))
    while kraft < one:                          # shorten the longest code, most frequent first
        m = max(range(n), key=lambda i: (ln[i], i))
        kraft += 1 << (HUF_MAX_BITS - ln[m])
        ln[m] -= 1
        if steps is not None:
            steps.append(("shrink", order[m][1]))
    return {s: ln[i] for i, (_, s) in enumerate(order)}


def huf_description(lengths):
    """The Huffman tree description of `lengths`, or None when encode.cuh cannot write one."""
    weights = E.huf_weights(lengths)
    nw = len(weights)
    if nw <= WEIGHTS_DIRECT_MAX:
        return E.write_huf_desc(weights, ("direct",))
    cnt = np.bincount(weights).tolist()
    if sum(1 for c in cnt if c) < 2:
        return None                             # every state would read 0 bits: the decoder could not find the end
    norm = fse_normalize(cnt, nw, WEIGHTS_LOG)
    body = E.huf_fse_weights(weights, WEIGHTS_LOG, norm, init_state)
    return bytes([len(body)]) + body if len(body) < 128 else None


def code_lengths(table):
    """{symbol: code length} of a huf_table."""
    mb, entries = table
    out = {}
    for s, nb in entries:
        out.setdefault(s, nb)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# FSE
# ---------------------------------------------------------------------------------------------------------------------------
def fse_normalize(cnt, total, log):
    """Normalized counts of cnt[0..maxsym] (last nonzero) summing to 2^log: -1 below one cell, else rounded to nearest and at
    least 1; a positive remainder goes to the first largest; a deficit is taken one cell at a time from the current maximum."""
    norm, used, best, largest = [], 0, -1, 0
    for s, c in enumerate(cnt):
        if not c:
            norm.append(0)
        elif (c << log) < total:
            norm.append(-1)
            used += 1
        else:
            v = max(1, ((c << log) + total // 2) // total)
            norm.append(v)
            used += v
            if v > best:
                best, largest = v, s
    diff = (1 << log) - used
    if diff > 0:
        norm[largest] += diff
    for _ in range(-diff):
        norm[norm.index(max(norm))] -= 1
    return norm


def fse_pick_log(n, maxsym, distinct, max_log):
    """FSE_optimalTableLog's rule, at least 5 and enough cells for `distinct` symbols."""
    log = max((n - 1).bit_length() - 1 - 2, 0) if n > 1 else 0
    log = min(log, max_log)
    min_log = min(n.bit_length(), maxsym.bit_length() + 1)
    log = max(log, min_log, 5)
    while (1 << log) < distinct:
        log += 1
    return min(log, max_log)


def init_state(tab, sym):
    """The state a chain of `sym` ends in: its first state in the table's index order (FSE_initCState on this spread)."""
    return E._first_state(tab, sym)


def log2_q8(p):
    """log2(p) in 8-bit fixed point, in integers: the integer part from the highest bit, the fraction by squaring the mantissa."""
    hb = p.bit_length() - 1
    x, r = (p << 16) >> hb, hb << 8
    for i in range(7, -1, -1):
        x = (x * x) >> 16
        if x >= 2 << 16:
            x >>= 1
            r |= 1 << i
    return r


def fse_cost_q8(cnt, norm, log):
    """Estimated bits (8-bit fixed point) of coding cnt with normalized counts norm at `log`; a -1 count costs as 1."""
    return sum(c * ((log << 8) - log2_q8(max(norm[s] if s < len(norm) else 0, 1))) for s, c in enumerate(cnt) if c)


# ---------------------------------------------------------------------------------------------------------------------------
# a formatted dictionary's tables
# ---------------------------------------------------------------------------------------------------------------------------
class Tables:
    """A formatted dictionary's entropy tables as the encoder uses them: the Huffman table and (log, norm) of LL / OF / ML."""

    def __init__(self, formatted):
        d = bytes(formatted)
        assert d[:4] == struct.pack("<I", 0xEC30A437)
        weights, used = E.read_huf_desc(d[8:])
        self.huf = E.huf_table(weights)
        self.huf_len = code_lengths(self.huf)
        p = 8 + used
        fse = {}
        for t in (OF, ML, LL):                  # the dictionary's order
            log, norm, used = E.read_ncount(d[p:])
            fse[t] = (log, norm)
            p += used
        self.fse = [fse[LL], fse[OF], fse[ML]]


# ---------------------------------------------------------------------------------------------------------------------------
# block
# ---------------------------------------------------------------------------------------------------------------------------
def raw_literals(lits):
    return E.lit_header(0, len(lits)) + lits


def literals_section(lits, tables=None):
    """(bytes, mode RAW / HUF / TREELESS) of the literals section."""
    n = len(lits)
    cnt = np.bincount(np.frombuffer(lits, dtype=np.uint8), minlength=256)
    raw = raw_literals(lits)
    best, mode = raw, RAW
    if n > RAW_LITERALS_MAX and np.count_nonzero(cnt) >= 2:
        lengths = huf_lengths(cnt)
        desc = huf_description(lengths)
        if desc is not None:
            pay = E.lit_payload(E.huf_table(E.huf_weights(lengths)), lits, 4)
            csize = len(desc) + len(pay)
            hsize = 4 if n < LIT_HEADER_4_MAX and csize < LIT_HEADER_4_MAX else 5
            if hsize + csize < n + 3:           # Huffman pays (compressed.rs:367-371)
                best, mode = E.lit_header(2, n, csize, 4, 2 if hsize == 4 else 3) + desc + pay, HUF
    if tables is not None and n >= 2 and all(tables.huf_len.get(s) for s in np.flatnonzero(cnt).tolist()):
        streams = 1 if n < TREELESS_1_STREAM else 4
        pay = E.lit_payload(tables.huf, lits, streams)
        if not (streams == 1 and len(pay) >= 1024):
            sf = 0 if streams == 1 else 2 if n < LIT_HEADER_4_MAX and len(pay) < LIT_HEADER_4_MAX else 3
            treeless = E.lit_header(3, n, len(pay), streams, sf) + pay
            if len(treeless) < len(best):
                best, mode = treeless, TREELESS
    return best, mode


def codes(recs):
    """LL, OF, ML codes of records (ll, ml, of) as numpy arrays; OF's is floor(log2(of + 3)) mod 2^32."""
    a = np.array(recs, dtype=np.int64).reshape(-1, 3)
    ofc = np.array([((of + 3) & 0xFFFFFFFF).bit_length() - 1 for _, _, of in recs], dtype=np.int64)
    return [np.searchsorted(LL_BASE, a[:, 0], side="right") - 1, ofc, np.searchsorted(ML_BASE, a[:, 1], side="right") - 1]


def sequences_section(recs, tables=None):
    """(bytes, [LL, OF, ML] modes; 0 each without sequences)."""
    n = len(recs)
    out = bytearray(E.seq_count(n))
    if not n:
        return bytes(out), [0, 0, 0]
    modes, descs, tabs = [], b"", []
    for t, c in enumerate(codes(recs)):
        cnt = np.bincount(c, minlength=MAX_SYM[t] + 1).tolist()
        present = [s for s, x in enumerate(cnt) if x]
        maxsym = present[-1]
        if len(present) == 1:
            modes.append(RLE_MODE)
            descs += bytes([maxsym])
            tabs.append(("rle", maxsym))
            continue
        cnt = cnt[:maxsym + 1]
        log = fse_pick_log(n, maxsym, len(present), MAX_LOG[t])
        norm = fse_normalize(cnt, n, log)
        desc = E.write_ncount(norm, log)
        if tables is not None:
            dlog, dnorm = tables.fse[t]
            if (all(s < len(dnorm) and dnorm[s] for s in present) and
                    fse_cost_q8(cnt, dnorm, dlog) <= (len(desc) << 11) + fse_cost_q8(cnt, norm, log)):
                modes.append(REPEAT_MODE)
                tabs.append(E.fse_table(dnorm, dlog))
                continue
        modes.append(FSE_MODE)
        descs += desc
        tabs.append(E.fse_table(norm, log))
    out.append((modes[LL] << 6) | (modes[OF] << 4) | (modes[ML] << 2))
    out += descs
    ovs = [(ll, ml, (of + 3) & 0xFFFFFFFF) for ll, ml, of in recs]
    out += E.seq_bitstream(ovs, tabs, init_state)
    return bytes(out), modes


def encode_block(lits, recs, tables=None):
    """Content of a Compressed block for literals and records: (bytes, literal mode, [LL, OF, ML] modes).  tables: a formatted
    dictionary's Tables when the block is its frame's first."""
    lsec, lmode = literals_section(bytes(lits), tables)
    ssec, modes = sequences_section(recs, tables)
    return lsec + ssec, lmode, modes


def block(data, lits, recs, tables=None):
    """(block type 0 Raw / 1 RLE / 2 Compressed, body) of a block of `data` whose parse gave lits and recs."""
    data = bytes(data)
    if data and data.count(data[:1]) == len(data):
        return 1, data[:1]
    content = encode_block(lits, recs, tables)[0]
    return (2, content) if len(content) < len(data) else (0, data)


# ---------------------------------------------------------------------------------------------------------------------------
# the dictionary writer (dict_format.cpp)
# ---------------------------------------------------------------------------------------------------------------------------
DS_LIT, DS_LL, DS_ML, DS_OF = 0, 256, 256 + 36, 256 + 36 + 53
NEAR_FLAT = {s: 7 if s == 0 else 9 if s >= 254 else 8 for s in range(256)}   # 2^-7 + 2 * 2^-9 = 3 * 2^-8


def scaled_counts(counts, need):
    """Counts shifted right until their total is below 2^30 - 512 (a nonzero count staying >= 1); every symbol <= need >= 1."""
    total = sum(int(c) for c in counts)
    shift = 0
    while (total >> shift) >= (1 << 30) - 512:
        shift += 1
    return [max(int(c) >> shift, 1 if c else 0, 1 if s <= need else 0) for s, c in enumerate(counts)]


def dict_header(counts, content_len):
    """The dictionary writer's header without magic and ID: Huffman description, OF / ML / LL descriptions (logs 8 / 9 / 9),
    repeat offsets 1, 4, 8."""
    lit = scaled_counts(counts[DS_LIT:DS_LIT + 256], 255)
    desc = huf_description(huf_lengths(lit))
    if desc is None:
        desc = huf_description(NEAR_FLAT)
    out = bytearray(desc)
    for lo, n, log, need in ((DS_OF, 32, 8, min(31, (content_len + 131072).bit_length() - 1)), (DS_ML, 53, 9, 52), (DS_LL, 36, 9, 35)):
        cnt = scaled_counts(counts[lo:lo + n], need)
        maxsym = max(s for s, c in enumerate(cnt) if c)
        cnt = cnt[:maxsym + 1]
        out += E.write_ncount(fse_normalize(cnt, sum(cnt), log), log)
    return bytes(out) + struct.pack("<3I", 1, 4, 8)


def dict_from_counts(counts, content, dict_id=0, dict_cap=None):
    """The formatted dictionary b200z_debug_dict_from_counts writes: header, then the content's last bytes that fit dict_cap;
    a zero dict_id is derived from those bytes as libzstd does (XXH64 mod (2^31 - 32768) + 32768)."""
    import cparse
    hdr = dict_header(counts, len(content))
    keep = len(content) if dict_cap is None else min(len(content), dict_cap - 8 - len(hdr))
    tail = bytes(content)[len(content) - keep:]
    if not dict_id:
        dict_id = cparse.xxh64(tail) % ((1 << 31) - 32768) + 32768
    return struct.pack("<II", 0xEC30A437, dict_id) + hdr + tail
