"""Crafted zstd frames with chosen entropy sections, shared by the CPU and GPU tests of the decoder's table builders (k_setup:
fse_build_warp / huf_build_warp in setup.cuh, the lane-0 parsers and the serial builders of tables.cuh) and literal streams (k_huf).

A Compressed block is written from an explicit entropy spec (`Blk`), not from what an encoder would choose: the Huffman code
length of every symbol and how its weights are described (direct, or FSE-compressed with given normalized counts and accuracy
log), 1 or 4 streams, the literals header's size format, Treeless literals; one mode per LL / OF / ML table (Predefined, RLE with a
code, FSE with given counts and log, Repeat).  The writer is plain Python; every table it encodes with is the reference's, so a
writer mistake shows up as a disagreement with the oracle and libzstd.

The reference is written from RFC 8878, independent of the oracle and of tables.cuh:
  fse_table(norm, log)  -- section 4.1.1: -1 symbols from the top down, spread step (size>>1)+(size>>3)+3, states numbered in
                           index order, nb / baseline of each state
  huf_table(weights)    -- section 4.2.1: max_bits, the implicit last weight, ranges longest code first and then by symbol
Frames follow seqcraft.frame's conventions (window log, content size, checksum); sequences are (ll, ml, Offset_Value) and the
content comes from seqcraft.execute.  `cases()` builds the crafted set; each id names the edge it sits on."""
import bisect
import random
import struct

import numpy as np

import seqcraft as S

ERROR = S.ERROR
MAX_LOG = {"ll": 9, "of": 8, "ml": 9}
MAX_SYM = {"ll": 35, "of": 31, "ml": 52}
KINDS = ("ll", "of", "ml")
# predefined distributions (RFC 8878 3.1.1.3.2.2)
PREDEF = {"ll": (6, [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1]),
          "ml": (6, [1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                            1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1]),
          "of": (5, [1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1])}
# code -> (baseline, extra bits) (RFC 8878 3.1.1.3.2.1.1)
LL_CODES = [(i, 0) for i in range(16)] + [(16, 1), (18, 1), (20, 1), (22, 1), (24, 2), (28, 2), (32, 3), (40, 3), (48, 4), (64, 6),
                                          (128, 7), (256, 8), (512, 9), (1024, 10), (2048, 11), (4096, 12), (8192, 13), (16384, 14),
                                          (32768, 15), (65536, 16)]
ML_CODES = [(i + 3, 0) for i in range(32)] + [(35, 1), (37, 1), (39, 1), (41, 1), (43, 2), (47, 2), (51, 3), (59, 3), (67, 4), (83, 4),
                                              (99, 5), (131, 7), (259, 8), (515, 9), (1027, 10), (2051, 11), (4099, 12), (8195, 13),
                                              (16387, 14), (32771, 15), (65539, 16)]


# ---------------------------------------------------------------------------------------------------------------------------
# reference tables
# ---------------------------------------------------------------------------------------------------------------------------
def fse_table(norm, log):
    """[(symbol, nb, baseline)] for every state of the FSE table of `norm` (-1 = "less than one") at accuracy `log`."""
    size = 1 << log
    sym = [None] * size
    high = size - 1
    for s, p in enumerate(norm):
        if p == -1:
            sym[high] = s
            high -= 1
    step, pos = (size >> 1) + (size >> 3) + 3, 0
    for s, p in enumerate(norm):
        for _ in range(max(p, 0)):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    assert pos == 0, "the counts do not add up to the table size"
    nxt = {s: (1 if p == -1 else p) for s, p in enumerate(norm) if p}
    out = []
    for s in sym:
        x = nxt[s]
        nxt[s] += 1
        nb = log - (x.bit_length() - 1)
        out.append((s, nb, (x << nb) - size))
    return out


def huf_weights(lengths):
    """Code lengths {symbol: length} (Kraft-complete) -> the weights a description lists (the last symbol's is implicit)."""
    mb = max(lengths.values())
    last = max(lengths)
    return [mb + 1 - lengths[s] if lengths.get(s) else 0 for s in range(last)]


def huf_table(weights):
    """(max_bits, [(symbol, nb)] * 2^max_bits) of the explicit `weights`; the implicit last symbol is len(weights), as u8."""
    total = sum(1 << (w - 1) for w in weights if w)
    mb = total.bit_length()
    left = (1 << mb) - total
    assert left & (left - 1) == 0, "leftover is not a power of two"
    full = list(weights) + [left.bit_length()]
    entries = []
    for nb in range(mb, 0, -1):
        for s, w in enumerate(full):
            if w and mb + 1 - w == nb:
                entries += [(s & 0xFF, nb)] * (1 << (mb - nb))
    return mb, entries


# ---------------------------------------------------------------------------------------------------------------------------
# bit writers / readers
# ---------------------------------------------------------------------------------------------------------------------------
class BitW:
    """Forward LSB-first bit writer; `backward()` closes a stream that is read from its end (marker bit, zero padding)."""

    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def add(self, v, nb):
        assert 0 <= v < (1 << nb) or (nb == 0 and v == 0)
        self.acc |= v << self.n
        self.n += nb
        while self.n >= 8:
            self.out.append(self.acc & 0xFF)
            self.acc >>= 8
            self.n -= 8

    def bytes(self):
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")

    def backward(self):
        self.add(1, 1)
        return self.bytes()


class FwdR:
    def __init__(self, data):
        self.v, self.pos, self.n = int.from_bytes(data, "little"), 0, len(data) * 8

    def get(self, nb):
        assert self.pos + nb <= self.n, "description truncated"
        r = (self.v >> self.pos) & ((1 << nb) - 1)
        self.pos += nb
        return r


def write_ncount(norm, log):
    """FSE table description (RFC 8878 4.1.1) of `norm`, which must end with a nonzero count."""
    w = BitW()
    w.add(log - 5, 4)
    size, counter, i = 1 << log, 0, 0
    while counter < size:
        p = norm[i]
        maxr = size - counter + 1
        bits = maxr.bit_length()
        lt, mask, value = (1 << bits) - 1 - maxr, (1 << (bits - 1)) - 1, p + 1
        if value < lt:
            w.add(value, bits - 1)
        elif value <= mask:
            w.add(value, bits)
        else:
            w.add(value + lt, bits)
        counter += 1 if p == -1 else p
        i += 1
        if p == 0:
            z = 0
            while i + z < len(norm) and norm[i + z] == 0:
                z += 1
            i += z
            while z >= 3:
                w.add(3, 2)
                z -= 3
            w.add(z, 2)
    assert i == len(norm), "counts after the table is full"
    return w.bytes()


def read_ncount(data):
    """(log, norm, bytes used) of an FSE table description: the plain reader the writer is checked against."""
    r = FwdR(data)
    log = r.get(4) + 5
    size, counter, norm = 1 << log, 0, []
    while counter < size:
        maxr = size - counter + 1
        bits = maxr.bit_length()
        lt, mask = (1 << bits) - 1 - maxr, (1 << (bits - 1)) - 1
        v = r.get(bits)
        if v & mask < lt:
            r.pos -= 1
            value = v & mask
        else:
            value = v - lt if v > mask else v
        p = value - 1
        norm.append(p)
        counter += 1 if p == -1 else p
        if p == 0:
            while True:
                z = r.get(2)
                norm += [0] * z
                if z != 3:
                    break
    return log, norm, (r.pos + 7) // 8


def _encoder(tab):
    """Encoding through the decoding table: {symbol: [state of the symbol whose [baseline, baseline + 2^nb) holds target, for
    every target in [0, 2^log)]} -- the ranges of one symbol's states cover the table exactly once."""
    enc = {}
    for x, (s, nb, base) in enumerate(tab):
        enc.setdefault(s, [None] * len(tab))[base:base + (1 << nb)] = [x] * (1 << nb)
    return enc


def _first_state(tab, sym, min_nb=0):
    return next(x for x, (s, nb, _) in enumerate(tab) if s == sym and nb >= min_nb)


def huf_fse_weights(weights, log, norm, first=_first_state):
    """The FSE-compressed form of a weight list (the description's body without its size byte): the table description, then
    two interleaved states, weight i from state i & 1.  first(tab, sym): the state a chain ends in (its symbol is decoded last);
    the update after weight n-2 reads past the stream's start, so that state needs nb >= 1."""
    tab, n = fse_table(norm, log), len(weights)
    assert n >= 2
    st = [None] * n
    st[n - 1] = first(tab, weights[n - 1])
    st[n - 2] = first(tab, weights[n - 2])
    assert tab[st[n - 2]][1] >= 1
    enc = _encoder(tab)
    for i in range(n - 3, -1, -1):
        st[i] = enc[weights[i]][st[i + 2]]
    w = BitW()
    for i in range(n - 3, -1, -1):
        _, nb, base = tab[st[i]]
        w.add(st[i + 2] - base, nb)
    w.add(st[1], log)
    w.add(st[0], log)
    return write_ncount(norm, log) + w.backward()


def write_huf_desc(weights, desc):
    """Huffman tree description: desc = ("direct",) or ("fse", log, norm)."""
    if desc[0] == "direct":
        n = len(weights)
        assert 1 <= n <= 128
        ws = list(weights) + [0]
        return bytes([127 + n]) + bytes((ws[i] << 4) | ws[i + 1] for i in range(0, n, 2))
    _, log, norm = desc
    body = huf_fse_weights(weights, log, norm, lambda tab, s: _first_state(tab, s, 1))
    assert len(body) < 128
    return bytes([len(body)]) + body


def read_huf_desc(data):
    """(weights, bytes used) of a Huffman tree description."""
    h = data[0]
    if h >= 128:
        n = h - 127
        return [(data[1 + i // 2] >> (0 if i & 1 else 4)) & 15 for i in range(n)], 1 + (n + 1) // 2
    log, norm, used = read_ncount(data[1:1 + h])
    tab = fse_table(norm, log)
    cs = data[1 + used:1 + h]
    v, p = int.from_bytes(cs, "little"), len(cs) * 8 - 8 + cs[-1].bit_length() - 1

    def get(nb):
        nonlocal p
        p -= nb
        return (v >> p) & ((1 << nb) - 1) if p >= 0 else (v & ((1 << (p + nb)) - 1)) << -p if p + nb > 0 else 0
    s = [get(log), get(log)]
    out, k = [], 0
    while True:
        out.append(tab[s[k]][0])
        _, nb, base = tab[s[k]]
        s[k] = base + get(nb)
        if p < 0:
            out.append(tab[s[1 - k]][0])
            return out, 1 + h
        k = 1 - k


# ---------------------------------------------------------------------------------------------------------------------------
# literals and sequences
# ---------------------------------------------------------------------------------------------------------------------------
class Huf:
    """A Huffman table to describe: code lengths {symbol: length} and the weight description ("direct",) / ("fse", log, norm)."""

    def __init__(self, lengths, desc=("direct",)):
        self.lengths, self.desc = dict(lengths), desc
        self.weights = huf_weights(self.lengths)
        self.table = huf_table(self.weights)

    def bytes(self):
        return write_huf_desc(self.weights, self.desc)


def huf_stream(table, data):
    """One Huffman stream: the codes of data's bytes from the last to the first, LSB first, then the end marker (packed with
    numpy: each code's bit j lands at the code's start + j)."""
    mb, entries = table
    code, ln = np.zeros(256, dtype=np.int64), np.zeros(256, dtype=np.int64)
    for i, (s, nb) in enumerate(entries):
        if not ln[s]:
            code[s], ln[s] = i >> (mb - nb), nb
    d = np.frombuffer(bytes(data), dtype=np.uint8)[::-1]
    c, n = code[d], ln[d]
    assert n.all(), "a byte without a code"
    start = np.cumsum(n) - n
    total = int(n.sum())
    bits = np.zeros(total + 1, dtype=np.uint8)
    for j in range(mb):
        m = n > j
        bits[start[m] + j] = (c[m] >> j) & 1
    bits[total] = 1
    return np.packbits(bits, bitorder="little").tobytes()


def lit_payload(table, data, streams):
    if streams == 1:
        return huf_stream(table, data)
    sz = (len(data) + 3) // 4
    parts = [huf_stream(table, data[k * sz:(k + 1) * sz]) for k in range(4)]
    return struct.pack("<3H", *(len(p) for p in parts[:3])) + b"".join(parts)


def lit_header(lt, regen, comp=None, streams=1, sf=None):
    if lt in (0, 1):
        if sf is None:
            sf = 0 if regen < 32 else (1 if regen < 4096 else 3)
        if sf in (0, 2):
            return bytes([lt | (sf << 2) | (regen << 3)])
        return (lt | (sf << 2) | (regen << 4)).to_bytes(2 if sf == 1 else 3, "little")
    if sf is None:
        m = max(regen, comp)
        sf = 0 if streams == 1 else (1 if m < 1024 else (2 if m < 16384 else 3))
    bits, n = {0: (10, 3), 1: (10, 3), 2: (14, 4), 3: (18, 5)}[sf]
    return (lt | (sf << 2) | (regen << 4) | (comp << (4 + bits))).to_bytes(n, "little")


LL_BASE = [b for b, _ in LL_CODES]
ML_BASE = [b for b, _ in ML_CODES]


def seq_codes(ll, ml, ov):
    llc = bisect.bisect_right(LL_BASE, ll) - 1
    mlc = bisect.bisect_right(ML_BASE, ml) - 1
    ofc = ov.bit_length() - 1
    return (llc, ll - LL_CODES[llc][0], LL_CODES[llc][1]), (ofc, ov - (1 << ofc), ofc), (mlc, ml - ML_CODES[mlc][0], ML_CODES[mlc][1])


def seq_count(n):
    """Number_of_Sequences in 1, 2 or 3 bytes."""
    return bytes([n]) if n < 128 else (bytes([(n >> 8) + 128, n & 0xFF]) if n < 0x7F00 else bytes([255]) + struct.pack("<H", n - 0x7F00))


def seq_bitstream(seqs, tabs, first=_first_state):
    """tabs: per kind (ll, of, ml) the decoding table, or ("rle", code).  first(tab, code): the state each chain ends in (the
    decoder's initial state; any state of the last sequence's code is legal)."""
    cs = [seq_codes(*q) for q in seqs]      # per sequence: ((llc, extra, nb), (ofc, ...), (mlc, ...))
    n = len(cs)
    states = [[None] * n for _ in range(3)]
    for k in range(3):
        if tabs[k][0] == "rle":
            assert all(c[k][0] == tabs[k][1] for c in cs), "a code other than the RLE code"
            continue
        enc, st = _encoder(tabs[k]), states[k]
        st[n - 1] = first(tabs[k], cs[n - 1][k][0])
        for i in range(n - 2, -1, -1):
            st[i] = enc[cs[i][k][0]][st[i + 1]]
    w = BitW()
    for i in range(n - 1, -1, -1):
        if i < n - 1:
            for k in (1, 2, 0):       # read as LL, ML, OF updates
                if tabs[k][0] != "rle":
                    _, nb, base = tabs[k][states[k][i]]
                    w.add(states[k][i + 1] - base, nb)
        for k in (0, 2, 1):           # read as OF, ML, LL extra bits
            w.add(cs[i][k][1], cs[i][k][2])
    for k in (2, 1, 0):               # read as LL, OF, ML initial states
        if tabs[k][0] != "rle":
            w.add(states[k][0], len(tabs[k]).bit_length() - 1)
    return w.backward()


class Blk:
    """One Compressed block.  lit: "huf" (new table `huf`), "treeless" (the frame's current table; `huf` only encodes a
    Treeless block that has none), "raw", "rle".  modes: per LL / OF / ML ("pre",), ("rle", code), ("fse", log, norm), ("rep",).
    raw: byte overrides for "huf_desc", "lit_payload", "seq_tables", "seq_bits" (error cases)."""

    def __init__(self, lits, lit="huf", huf=None, streams=4, sf=None, seqs=(), modes=None, raw=None):
        self.lits, self.lit, self.huf, self.streams, self.sf = bytes(lits), lit, huf, streams, sf
        self.seqs = list(seqs)
        self.modes = list(modes or [("pre",)] * 3)
        self.raw = raw or {}


def _mode_table(kind, m, cur):
    if m[0] == "pre":
        log, norm = PREDEF[kind]
        return fse_table(norm, log), {"log": log, "is_rle": 0, "entries": fse_table(norm, log)}
    if m[0] == "rle":
        return ("rle", m[1]), {"log": 0, "is_rle": 1, "entries": [(m[1], 0, 0)]}
    if m[0] == "fse":
        t = fse_table(m[2], m[1])
        return t, {"log": m[1], "is_rle": 0, "entries": t}
    return cur


def block_content(b, state):
    """Bytes of Compressed block `b`; updates `state` (the frame's current tables) and returns (content, its tables as the
    decoder should resolve them: {"huf", "ll", "of", "ml"} -> reference table or None)."""
    out, tabs = bytearray(), {"huf": None, "ll": None, "of": None, "ml": None}
    if b.lit in ("raw", "rle"):
        out += lit_header(0 if b.lit == "raw" else 1, len(b.lits), sf=b.sf)
        out += b.lits if b.lit == "raw" else b.lits[:1]
    else:
        if b.lit == "huf":
            desc = b.raw.get("huf_desc", b.huf.bytes() if b.huf else b"")
            if b.huf:
                state["huf"] = b.huf.table
        else:
            desc = b""
        table = state["huf"] or (b.huf.table if b.huf else None)
        tabs["huf"] = state["huf"]
        pay = b.raw["lit_payload"] if "lit_payload" in b.raw else lit_payload(table, b.lits, b.streams)
        out += lit_header(2 if b.lit == "huf" else 3, len(b.lits), len(desc) + len(pay), b.streams, b.sf) + desc + pay
    n = len(b.seqs)
    out += seq_count(n)
    if n:
        out.append(sum({"pre": 0, "rle": 1, "fse": 2, "rep": 3}[m[0]] << (6 - 2 * k) for k, m in enumerate(b.modes)))
        enc = []
        for k, kind in enumerate(KINDS):
            m = b.modes[k]
            if m[0] == "fse":
                out += write_ncount(m[2], m[1]) if "seq_tables" not in b.raw else b""
            elif m[0] == "rle" and "seq_tables" not in b.raw:
                out.append(m[1])
            if "seq_bits" in b.raw:
                continue
            got = _mode_table(kind, m, state[kind])
            if got is None and len(m) > 1:        # Repeat with nothing to repeat: encode with the given fallback table
                got = _mode_table(kind, m[1], None)
            elif got is not None:
                state[kind] = got
                tabs[kind] = got[1]
            enc.append(got[0] if got else None)
        out += b.raw.get("seq_tables", b"")
        out += b.raw["seq_bits"] if "seq_bits" in b.raw else seq_bitstream(b.seqs, enc)
    return bytes(out), tabs


def plain_blocks(blocks):
    return [("cmp", b.lits, b.seqs) if isinstance(b, Blk) else b for b in blocks]


def frame(blocks, window_log=17, checksum=True, dict_id=None, dict_state=None):
    """(frame bytes, per block: reference tables of a Compressed block or None).  Raw / RLE blocks as in seqcraft.frame."""
    plain = S.execute(plain_blocks(blocks), ov=True)
    fhd = (4 if checksum else 0) | (2 if dict_id is not None else 0)
    fcs = b""
    if plain is not ERROR:
        fcs = struct.pack("<I", len(plain))
        fhd |= 2 << 6
    out = struct.pack("<IBB", 0xFD2FB528, fhd, (window_log - 10) << 3) + (struct.pack("<H", dict_id) if dict_id is not None else b"") + fcs
    state = dict(dict_state or {"huf": None, "ll": None, "of": None, "ml": None})
    tabs = []
    for i, b in enumerate(blocks):
        last = 1 if i + 1 == len(blocks) else 0
        if isinstance(b, Blk):
            content, t = block_content(b, state)
            assert len(content) <= S.BLOCK_MAX
            out += struct.pack("<I", last | (2 << 1) | (len(content) << 3))[:3] + content
            tabs.append(t)
        elif b[0] == "raw":
            out += struct.pack("<I", last | (len(b[1]) << 3))[:3] + bytes(b[1])
            tabs.append(None)
        else:
            out += struct.pack("<I", last | (1 << 1) | (b[2] << 3))[:3] + bytes([b[1]])
            tabs.append(None)
    if checksum:
        from oracle import oracle as O
        out += struct.pack("<I", O.xxh64(plain if plain is not ERROR else b"") & 0xFFFFFFFF)
    return out, tabs


# ---------------------------------------------------------------------------------------------------------------------------
# formatted dictionaries (RFC 8878 5)
# ---------------------------------------------------------------------------------------------------------------------------
def dictionary(dict_id, huf, of, ml, ll, reps, content):
    """A formatted dictionary: Huffman description, FSE descriptions of OF / ML / LL ((log, norm) each), repeat offsets,
    content.  Returns (bytes, the tables a frame that uses it starts with)."""
    raw = (struct.pack("<II", 0xEC30A437, dict_id) + huf.bytes() + write_ncount(of[1], of[0]) + write_ncount(ml[1], ml[0]) +
           write_ncount(ll[1], ll[0]) + struct.pack("<3I", *reps) + bytes(content))
    st = {"huf": huf.table}
    for kind, (log, norm) in (("ll", ll), ("of", of), ("ml", ml)):
        st[kind] = (fse_table(norm, log), {"log": log, "is_rle": 0, "entries": fse_table(norm, log)})
    return raw, st


# ---------------------------------------------------------------------------------------------------------------------------
# the crafted cases
# ---------------------------------------------------------------------------------------------------------------------------
class Case:
    """One crafted frame.  error: the frame is invalid (a table or stream error the LZ77 reference cannot see).  libzstd: whether
    libzstd is expected to agree (it rejects a few things the reference accepts).  dict_raw: a formatted dictionary."""

    def __init__(self, group, name, blocks, error=False, libzstd=True, dict_raw=None, dict_id=None, dict_state=None, dict_descs=(),
                 window_log=17):
        self.group, self.id = group, f"{group}-{name}"
        self.dict_descs = list(dict_descs)
        self.blocks, self.libzstd, self.dict_raw = blocks, libzstd, dict_raw
        self.frame, self.tables = frame(blocks, window_log, dict_id=dict_id, dict_state=dict_state)
        # dictionary cases start with their repeat offsets at [1, 4, 8] and never reach into the dictionary's content
        self.expected = ERROR if error else S.execute(plain_blocks(blocks), ov=True)
        self.valid = self.expected is not ERROR
        self.cap = len(self.expected) if self.valid else max(1, S.nominal_size(plain_blocks(blocks)))

    def descriptions(self):
        """Every table description the frame (and its dictionary) carries: ("huf", Huf) and (kind, log, norm)."""
        out = list(self.dict_descs)
        for b in self.blocks:
            if isinstance(b, Blk):
                if b.lit == "huf" and b.huf and "huf_desc" not in b.raw:
                    out.append(("huf", b.huf))
                if b.seqs and "seq_tables" not in b.raw:
                    out += [(kind, m[1], m[2]) for kind, m in zip(KINDS, b.modes) if m[0] == "fse"]
        return out

    def __repr__(self):
        return self.id


def lengths_for(rng, syms, mb):
    """Kraft-complete code lengths over `syms` (>= mb + 1 of them, or 2 for mb = 1) with longest code exactly mb."""
    syms = list(syms)
    assert len(syms) <= 1 << mb
    keep = set(rng.sample(syms, 2))
    for attempt in range(8):            # random shortening, and as the last resort always the largest step that fits
        ln = {s: mb for s in syms}
        deficit = (1 << mb) - len(syms)
        while deficit:
            cand = [s for s in syms if s not in keep and ln[s] > 1 and 1 << (mb - ln[s]) <= deficit]
            if not cand:
                break
            big = max(1 << (mb - ln[s]) for s in cand)
            pool = [s for s in cand if 1 << (mb - ln[s]) == big] if attempt == 7 or rng.random() < 0.7 else cand
            s = rng.choice(pool)
            deficit -= 1 << (mb - ln[s])
            ln[s] -= 1
        if not deficit:
            return ln
    raise AssertionError("no complete code with these constraints")


def literals(rng, lengths, n):
    syms = sorted(lengths)
    w = [2.0 ** -lengths[s] for s in syms]
    out = bytearray(rng.choices(syms, w, k=n))
    for i, s in enumerate(syms[:n]):            # every symbol appears when there is room
        out[rng.randrange(n)] = s
    return bytes(out)


def rand_norm(rng, n, log, neg=0, zero_frac=0.0, keep=()):
    """Normalized counts over n symbols summing to 2^log (-1 counts 1), last one nonzero, `neg` of them -1."""
    size = 1 << log
    nz = [s for s in range(n) if s == n - 1 or s in keep or rng.random() >= zero_frac]
    assert len(nz) <= size
    negs = set(rng.sample([s for s in nz if s not in keep], min(neg, len(nz) - 1)))
    p = [0] * n
    pos = [s for s in nz if s not in negs]
    for s in nz:
        p[s] = -1 if s in negs else 1
    for _ in range(size - len(nz)):
        p[rng.choice(pos)] += 1
    return p


USABLE = {"ll": 24, "of": 16, "ml": 42}   # highest code the generated sequences use (keeps blocks small)


def gen_seqs(rng, n, codes, pos):
    """n sequences whose LL / OF / ML codes come from codes[kind] (lists), starting at output position pos (>= 8)."""
    seqs = []
    for _ in range(n):
        llc, mlc = rng.choice(codes["ll"]), rng.choice(codes["ml"])
        ofc = rng.choice([c for c in codes["of"] if c < 2 or (1 << c) - 3 <= pos])
        ll = LL_CODES[llc][0] + rng.randrange(1 << LL_CODES[llc][1])
        ml = ML_CODES[mlc][0] + rng.randrange(1 << ML_CODES[mlc][1])
        if ofc == 0:
            ov = 1
        elif ofc == 1:
            ov = 2
        else:
            lo = 1 << ofc
            ov = lo + rng.randrange(min(lo, pos + ll + 3 - lo + 1))
            assert 4 <= ov and ov - 3 <= pos + ll
        seqs.append((ll, ml, ov))
        pos += ll + ml
    return seqs


def codes_of(modes, state=None):
    out = {}
    for kind, m in zip(KINDS, modes):
        if m[0] == "rle":
            out[kind] = [m[1]]
        elif m[0] == "fse":
            out[kind] = [s for s, p in enumerate(m[2]) if p and s <= USABLE[kind]]
        elif m[0] == "pre":
            out[kind] = [s for s, p in enumerate(PREDEF[kind][1]) if p and s <= USABLE[kind]]
        elif len(m) > 1:
            out[kind] = codes_of([m[1]] * 3)[kind]
        else:
            out[kind] = state[kind]
    return out


def prefix(rng, n=64):
    return ("raw", bytes(rng.randrange(256) for _ in range(n)))


def _size(seqs):
    return sum(q[0] for q in seqs)


def seq_block(rng, modes, nseq=60, pos=64, lit_mode="raw", huf=None, codes=None, tail=3):
    c = codes or codes_of(modes)
    seqs = gen_seqs(rng, nseq, c, pos)
    lits = bytes(rng.randrange(256) for _ in range(_size(seqs) + tail)) if lit_mode == "raw" else literals(rng, huf.lengths, _size(seqs) + tail)
    return Blk(lits, lit_mode, huf=huf, seqs=seqs, modes=modes)


def huf_tables(rng):
    out = []
    for mb in range(1, 12):                                   # max_bits 1-11
        n = 2 if mb == 1 else rng.randint(mb + 1, min(1 << mb, 256))
        ln = lengths_for(rng, rng.sample(range(256), n), mb)
        h = Huf(ln) if max(ln) <= 128 else fse_weights(rng, ln, 6)
        out.append(Case("huf-tables", f"max_bits{mb}", [Blk(literals(rng, h.lengths, 400), huf=h, streams=rng.choice((1, 4)))]))
    for n in (2, 31, 32, 33, 64, 65, 96, 97, 128, 129, 200, 255, 256):   # symbol counts across huf_build_warp's 32-lane chunks
        mb = max(11 if n > 128 else 8, (n - 1).bit_length()) if n > 2 else 1
        h = fse_weights(rng, lengths_for(rng, range(n), mb), 6) if n > 129 else Huf(lengths_for(rng, range(n), mb))
        out.append(Case("huf-tables", f"nsym{n}-max_bits{h.table[0]}", [Blk(literals(rng, h.lengths, 1500), huf=h)]))
    h = fse_weights(rng, {0: 1, 255: 1}, 5)                  # 254 zero weights between them
    out.append(Case("huf-tables", "sparse-0-and-255", [Blk(literals(rng, h.lengths, 300), huf=h)]))
    h = fse_weights(rng, lengths_for(rng, rng.sample(range(255), 40) + [255], 9), 6)
    out.append(Case("huf-tables", "implicit-last-255", [Blk(literals(rng, h.lengths, 900), huf=h)]))
    for nw in (1, 2, 15, 16, 127, 128):                       # direct weights: odd counts and the final nibble
        mb = 1 if nw == 1 else max(2, nw.bit_length())
        syms = list(range(nw + 1)) if nw > 1 else [0, 1]
        h = Huf(lengths_for(rng, syms, mb) if nw > 1 else {0: 1, 1: 1})
        assert len(h.weights) == nw
        out.append(Case("huf-tables", f"direct-{nw}-weights", [Blk(literals(rng, h.lengths, 700), huf=h)]))
    for log in (5, 6):                                        # FSE-compressed weights: either state may end
        for neg in (0, 1):
            for nw in (40, 41):
                h = fse_weights(rng, lengths_for(rng, range(nw + 1), 10), log, neg)
                assert len(h.weights) == nw
                out.append(Case("huf-tables", f"fse-weights-log{log}-neg{neg}-{nw}-weights", [Blk(literals(rng, h.lengths, 600), huf=h)]))
    return out


def fse_weights(rng, lengths, log, neg=0):
    """A Huffman table for `lengths` whose weights are described FSE-compressed at accuracy `log`."""
    return Huf(lengths, ("fse", log, _weight_norm(rng, huf_weights(lengths), log, neg)))


def _weight_norm(rng, weights, log, neg=0):
    """Normalized counts over the weight values a description uses (each used value nonzero; zero runs where unused)."""
    used = sorted(set(weights))
    n = max(used) + 1
    size = 1 << log
    p = [0] * n
    negs = set(rng.sample(used, min(neg, len(used) - 1)))
    for w in used:
        p[w] = -1 if w in negs else 1
    pos = [w for w in used if w not in negs]
    for _ in range(size - len(used)):
        p[rng.choice(pos)] += 1
    return p


def huf_streams(rng):
    out = []
    h = Huf(lengths_for(rng, range(60), 9))
    for regen in (1, 2, 1022, 1023):                          # one stream, the 10-bit size format's edge
        out.append(Case("huf-streams", f"1stream-regen{regen}", [Blk(literals(rng, h.lengths, regen), huf=h, streams=1)]))
    for regen in range(1, 17):                                # 4 streams: regen < 3*S takes the exact path; regen 6 leaves stream 3 empty
        out.append(Case("huf-streams", f"4streams-regen{regen}", [Blk(literals(rng, h.lengths, regen), huf=h, streams=4)],
                        libzstd=regen >= 6))
    blocks = [prefix(rng, 16)]
    for r in range(16):                                       # dst + k*S at every residue mod 16
        blocks.append(Blk(literals(rng, h.lengths, 4 * (64 + r)), huf=h))
    out.append(Case("huf-streams", "dst+k*S-every-residue16", blocks))
    for r in range(16):                                       # stream starts at every residue mod 16 (PosRing's gm1)
        out.append(Case("huf-streams", f"stream-start-residue{r}", [prefix(rng, r + 1), Blk(literals(rng, h.lengths, 3000), huf=h)]))
    flat = Huf({s: 7 for s in range(128)})                    # 7-bit codes: k symbols make a stream of ceil((7k + 1) / 8) bytes
    for ln in (127, 128, 129, 144):
        k = (8 * ln - 1) // 7
        out.append(Case("huf-streams", f"stream-bytes{ln}", [Blk(bytes(rng.randrange(128) for _ in range(4 * k)), huf=flat)]))
    h1 = Huf({0: 1, 1: 1})
    out.append(Case("huf-streams", "131072-literals-max_bits1", [Blk(bytes(rng.randrange(2) for _ in range(S.BLOCK_MAX)), huf=h1)]))
    h11 = fse_weights(rng, lengths_for(rng, range(256), 11), 6)
    out.append(Case("huf-streams", "131072-literals-max_bits11", [Blk(literals(rng, h11.lengths, S.BLOCK_MAX - 8), huf=h11)]))
    # every literal an 11-bit code: 44 bits per window of four symbols, the most the fast path's ring has to keep up with
    long11 = [s for s, n in h11.lengths.items() if n == 11]
    out.append(Case("huf-streams", "90000-literals-all-11-bit-codes", [Blk(bytes(rng.choices(long11, k=90000)), huf=h11)]))
    blocks = []
    for mb in (11, 2, 7, 1, 9, 4, 10, 6):                     # eight max_bits side by side in one k_huf CTA
        hh = Huf(lengths_for(rng, range(mb + 1 if mb > 1 else 2), mb))
        blocks.append(Blk(literals(rng, hh.lengths, rng.randint(200, 3000)), huf=hh))
    out.append(Case("huf-streams", "8-max_bits-in-one-cta", blocks))
    return out


def treeless(rng):
    out = []
    h = Huf(lengths_for(rng, range(50), 8))
    h2 = Huf(lengths_for(rng, range(30, 120), 10))
    L = lambda n, hh=h: literals(rng, hh.lengths, n)
    out.append(Case("treeless", "after-compressed", [Blk(L(500), huf=h), Blk(L(700), "treeless")]))
    out.append(Case("treeless", "chain-of-4", [Blk(L(500), huf=h)] + [Blk(L(300 + 100 * i), "treeless", streams=1 + 3 * (i & 1)) for i in range(4)]))
    out.append(Case("treeless", "after-raw-rle-literals", [Blk(L(500), huf=h), Blk(b"rawlits", "raw"), Blk(b"\x07" * 40, "rle"), Blk(L(900), "treeless")]))
    out.append(Case("treeless", "after-raw-rle-blocks", [Blk(L(500), huf=h), ("raw", b"x" * 100), ("rle", 3, 50), Blk(L(900), "treeless")]))
    out.append(Case("treeless", "after-new-table", [Blk(L(500), huf=h), Blk(L(400, h2), huf=h2), Blk(L(600, h2), "treeless")]))
    b0 = seq_block(rng, [("pre",)] * 3, lit_mode="huf", huf=h)
    b1 = seq_block(rng, [("rep",)] * 3, pos=64 + S.nominal_size([("cmp", b0.lits, b0.seqs)]), lit_mode="treeless", huf=h,
                   codes=codes_of([("pre",)] * 3))
    out.append(Case("treeless", "with-sequences", [prefix(rng), b0, b1]))
    out.append(Case("treeless", "first-use-error", [Blk(L(300), "treeless", huf=h)], error=True))
    out.append(Case("treeless", "after-frame-with-table", [Blk(L(300, h2), huf=h2)]))
    out.append(Case("treeless", "next-frame-starts-treeless-error", [Blk(L(300, h2), "treeless", huf=h2)], error=True))
    return out


def fse_tables(rng):
    out = []
    for kind in KINDS:
        k = KINDS.index(kind)
        top = MAX_SYM[kind]

        def case(name, m, nseq=80):
            modes = [("pre",)] * 3
            modes[k] = m
            out.append(Case("fse-tables", f"{kind}-{name}", [prefix(rng, 70000 if kind == "of" else 64), seq_block(rng, modes, nseq, pos=70000 if kind == "of" else 64)]))
        for log in range(5, MAX_LOG[kind] + 1):
            case(f"log{log}", ("fse", log, rand_norm(rng, min(top + 1, 20 + log), log, neg=2, zero_frac=0.2, keep=(3,))))
        log = MAX_LOG[kind]
        case(f"ends-at-top-symbol{top}", ("fse", log, rand_norm(rng, top + 1, log, neg=3, zero_frac=0.3, keep=(2, 5))))
        for n in (31, 32, 33):
            if n <= top + 1:
                case(f"nsym{n}", ("fse", 6, rand_norm(rng, n, 6, neg=1, keep=(4,))))
        case("no-neg", ("fse", 7, rand_norm(rng, 25, 7, keep=(6,))))
        case("one-neg", ("fse", 7, rand_norm(rng, 25, 7, neg=1, keep=(6,))))
        case("neg-on-most-cells", ("fse", 5, [-1 if s != 7 else 2 for s in range(31)]))   # 30 of 32 cells "less than one"
        for log in (5, MAX_LOG[kind]):
            case(f"single-symbol-log{log}", ("fse", log, [0] * 9 + [1 << log]), nseq=40)
        big = (1 << 8) - 8 - 9 - 10 - 1
        case("own-big-8-9-cells", ("fse", 8, [8, 9, 0, 0, big, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1]))
        # zero runs: 3 + 3 + ... chained flags, and runs of 25+ zeros (the 24-zero form of an encoder)
        zr = {"ll": [30, 2] + [0] * 30 + [32], "of": [0, 0, 0, 30, 2] + [0] * 25 + [32], "ml": [30, 2] + [0] * 40 + [32]}[kind]
        case(f"zero-run{max(len(g) for g in _runs(zr))}", ("fse", 6, zr))
        case("rle-code0", ("rle", 0))
        case("predefined", ("pre",))
    # RLE with the top codes: LL 35 (>= 65536 literals per sequence), ML 52 (matches of >= 65539); OF 31 cannot be valid
    lits = bytes(rng.randrange(256) for _ in range(65536 + 8))
    out.append(Case("fse-tables", "ll-rle-top-code35", [prefix(rng), Blk(lits, "raw", seqs=[(65536, 5, 10)], modes=[("rle", 35), ("pre",), ("pre",)])]))
    out.append(Case("fse-tables", "ml-rle-top-code52", [prefix(rng), Blk(b"abcd", "raw", seqs=[(4, 65539 + 77, 12)], modes=[("pre",), ("pre",), ("rle", 52)])]))
    out.append(Case("fse-tables", "of-rle-top-code31-offset-error", [prefix(rng), Blk(b"abcd", "raw", seqs=[(4, 5, (1 << 31) + 5)], modes=[("pre",), ("rle", 31), ("pre",)])]))
    return out


def _runs(norm):
    run = []
    for p in norm:
        if p == 0:
            run.append(p)
        elif run:
            yield run
            run = []
    if run:
        yield run


def repeats(rng):
    out = []
    fse = lambda kind, log: ("fse", log, rand_norm(rng, 20, log, neg=1, keep=(2, 3, 4)))
    defs = {"fse": [fse("ll", 6), fse("of", 5), fse("ml", 7)], "rle": [("rle", 4), ("rle", 6), ("rle", 9)], "pre": [("pre",)] * 3}
    seps = {"none": [], "raw": [("raw", b"q" * 40)], "rle": [("rle", 0x33, 70)], "noseq": [Blk(b"0123", "raw")]}
    for d, modes in defs.items():
        for sep, mid in seps.items():
            if d != "fse" and sep != "none":
                continue
            b0 = seq_block(rng, modes, 50)
            pos = 64 + S.nominal_size([("cmp", b0.lits, b0.seqs)]) + S.nominal_size(plain_blocks(mid))
            b1 = seq_block(rng, [("rep",)] * 3, 70, pos=pos, codes=codes_of(modes))
            out.append(Case("repeat", f"after-{d}-across-{sep}", [prefix(rng), b0] + mid + [b1]))
    b0 = seq_block(rng, defs["fse"], 50)
    mixed = [("fse", 7, rand_norm(rng, 22, 7, neg=2, keep=(3,))), ("rep",), ("rle", 5)]
    c = codes_of(mixed, {"of": codes_of(defs["fse"])["of"]})
    b1 = seq_block(rng, mixed, 60, pos=64 + S.nominal_size([("cmp", b0.lits, b0.seqs)]), codes=c)
    b2 = seq_block(rng, [("rep",), ("pre",), ("rep",)], 40, pos=64 + S.nominal_size(plain_blocks([b0, b1])),
                   codes={"ll": c["ll"], "of": codes_of([("pre",)] * 3)["of"], "ml": [5]})
    out.append(Case("repeat", "mixed-ll-fse-of-rep-ml-rle", [prefix(rng), b0, b1, b2]))
    for k, kind in enumerate(KINDS):
        modes = [("pre",)] * 3
        modes[k] = ("rep", ("pre",))
        out.append(Case("repeat", f"{kind}-first-use-error", [prefix(rng), seq_block(rng, modes, 20)], error=True))
    return out


def errors(rng):
    out = []
    pre = [("pre",)] * 3
    bits = b"\x5a\x3c\x99\x01"

    def seqerr(name, modes, tables):
        b = seq_block(rng, pre, 10)
        b.modes, b.raw = modes, {"seq_tables": tables, "seq_bits": bits}
        out.append(Case("errors", name, [prefix(rng), b], error=True))
    for k, kind in enumerate(KINDS):
        m = list(pre)
        m[k] = ("fse", 0, None)
        seqerr(f"{kind}-acc-log{MAX_LOG[kind] + 1}", m, bytes([MAX_LOG[kind] + 1 - 5, 0xFF, 0xFF, 0xFF]))
        n = MAX_SYM[kind] + 2
        seqerr(f"{kind}-too-many-symbols{n}", m, write_ncount([1] * (n - 1) + [64 - n + 1], 6))
        seqerr(f"{kind}-truncated-description", m, write_ncount(rand_norm(rng, 20, 7, neg=2), 7)[:5])
        m[k] = ("rle", 0)
        seqerr(f"{kind}-rle-code{MAX_SYM[kind] + 1}", m, bytes([MAX_SYM[kind] + 1]))
    h = Huf(lengths_for(rng, range(20), 6))
    lits = literals(rng, h.lengths, 200)

    def huferr(name, desc=None, payload=None, streams=4, libzstd=True):
        raw = {}
        if desc is not None:
            raw["huf_desc"] = desc
        if payload is not None:
            raw["lit_payload"] = payload
        out.append(Case("errors", name, [Blk(lits, huf=h, streams=streams, raw=raw)], error=True, libzstd=libzstd))
    huferr("huf-weight12", bytes([127 + 3, 0x1C, 0x10]))
    huferr("huf-leftover-not-pow2", bytes([127 + 4, 0x21, 0x11]))
    huferr("huf-max-bits12", bytes([127 + 2, 0xBB]))
    good = h.bytes() if h.desc[0] == "fse" else Huf(h.lengths, ("fse", 6, _weight_norm(rng, h.weights, 6))).bytes()
    _, _, used = read_ncount(good[1:])
    huferr("huf-fse-header-uses-too-many-bytes", bytes([used - 1]) + good[1:])
    huferr("huf-fse-header-too-few-bytes", bytes([127]) + good[1:], payload=b"", streams=1)
    pay = lit_payload(h.table, lits, 4)
    huferr("jump-table-5-bytes", payload=pay[:5])
    huferr("streams-past-payload", payload=struct.pack("<3H", 200, 200, 200) + pay[6:])
    huferr("empty-stream", payload=struct.pack("<3H", 0, 0, 0) + pay[6:])
    huferr("empty-single-stream", payload=b"", streams=1)
    huferr("stream-last-byte-zero", payload=lit_payload(h.table, lits, 1) + b"\x00", streams=1)
    return out


def dict_cases(rng):
    h = fse_weights(rng, lengths_for(rng, range(256), 11), 6, 1)
    of =(8, rand_norm(rng, 20, 8, neg=4, keep=(2, 3, 4, 5)))
    ml = (7, rand_norm(rng, 30, 7, neg=2, keep=(0, 1, 2)))
    ll = (6, rand_norm(rng, 22, 6, neg=1, keep=(0, 1, 2)))
    raw, st = dictionary(0x1234, h, of, ml, ll, (1, 4, 8), bytes(rng.randrange(256) for _ in range(300)))
    codes = {"ll": [s for s in range(22) if ll[1][s]], "of": [s for s in range(2, 7) if of[1][s]], "ml": [s for s in range(30) if ml[1][s]]}
    b0 = seq_block(rng, [("rep",)] * 3, 80, pos=64, lit_mode="treeless", huf=h, codes=codes)
    b1 = seq_block(rng, [("rep",)] * 3, 40, pos=64 + S.nominal_size([("cmp", b0.lits, b0.seqs)]), lit_mode="treeless", huf=h, codes=codes)
    return [Case("dict", "treeless-and-repeat-from-dictionary", [prefix(rng), b0, b1], dict_raw=raw, dict_id=0x1234, dict_state=st,
                 dict_descs=[("huf", h), ("of",) + of, ("ml",) + ml, ("ll",) + ll])]


GROUPS = {"huf-tables": huf_tables, "huf-streams": huf_streams, "treeless": treeless, "fse-tables": fse_tables, "repeat": repeats,
          "errors": errors, "dict": dict_cases}


def cases(group=None):
    """The crafted cases (all groups, or one), built from fixed seeds."""
    out = []
    for i, (g, fn) in enumerate(GROUPS.items()):
        if group is None or g == group:
            out += fn(random.Random(0xE7C0 + i))
    return out


def oracle_decode(oracle, c):
    """Decodes case `c` with the oracle; checks its trace literals and sequences against what was requested (up to where it
    stopped).  Returns (content, None) or (None, (error leaf, stage))."""
    d = oracle.FrameDecoder()
    d.trace_enable()
    if c.dict_raw is not None:
        d.add_dict(c.dict_raw)
    try:
        r = d.reset(c.frame)
        d.decode_blocks(r, oracle.ALL)
        res = (d.collect(), None)
    except oracle.OracleError as e:
        res = (None, (oracle.error_names()[e.code].replace("ZO_", ""), e.stage))
    _, lits, seqs = d.trace()
    cmp = [b for b in c.blocks if isinstance(b, Blk)]
    want_l = b"".join(b.lits for b in cmp)
    want_s = [q for b in cmp for q in b.seqs]
    got_s = [tuple(int(x) for x in s[:3]) for s in seqs]
    assert lits == want_l[:len(lits)], "the oracle decoded other literals than the ones requested"
    assert got_s == want_s[:len(got_s)], "the oracle decoded other sequences than the ones requested"
    if res[1] is None:
        assert lits == want_l and got_s == want_s
    return res
