"""Crafted frames that reach past the decoder's buffer: into a dictionary, or beyond the window.  Shared by the CPU and GPU tests.

`execute` is the model: DecodeBuffer::repeat / repeat_from_dict (decode_buffer.rs:79-179) and execute_sequences
(sequence_execution.rs) restated in plain Python, independent of the oracle and of the kernels.  Two of the reference's rules
are not the format's, and this project keeps them:
  * an offset is checked against the undrained buffer (produced - drained), not against the window;
  * the dictionary can be reached only while total_output_counter <= window_size.  Literals and in-buffer matches advance that
    counter; Raw and RLE blocks and a match copied wholly from the dictionary do not.
`execute(..., rfc=True)` is the RFC 8878 reading instead: an offset is valid iff it is at most produced + dictionary length and
at most the window, and a formatted dictionary's repeat offsets must lie in [1, content length] (as libzstd requires).  A case
marked `quirk` is one where the two readings differ.  The RFC reading covers offsets only: it leaves out Block_Maximum_Size
(min(Window_Size, 128 KiB)), which the cases with a small window and larger Raw, RLE or Compressed blocks exceed.  Those cases are
quirk or error cases, so no comparison with libzstd depends on the limit.

Frames use Offset_Value mode (seqcraft `ov=True`): 1-3 are repeat codes, a new offset o is written as o + 3.  Blocks are as in
seqcraft: ("raw", bytes), ("rle", byte, count), ("cmp", literals, [(ll, ml, offset_value), ...])."""
import os
import random
import struct

import seqcraft as S

ERROR = S.ERROR
HERE = os.path.dirname(os.path.abspath(__file__))
EXEC_BATCH, FSE_PUBLISH, FSE_FAST_XBITS, WHY_SEQ_CHECK = S.EXEC_BATCH, S.FSE_PUBLISH, S.FSE_FAST_XBITS, S.WHY_SEQ_CHECK
STAGE_EXECUTE, STAGE_DRAIN = 6, 9
NOT_IN_DICT, TOO_BIG = "ERR_EXEC_NOT_ENOUGH_BYTES_IN_DICTIONARY", "ERR_EXEC_OFFSET_TOO_BIG"


# ---------------------------------------------------------------------------------------------------------------------------
# dictionaries
# ---------------------------------------------------------------------------------------------------------------------------
def _golden_tables():
    """The Huffman and FSE table section of the golden dictionary (tests/golden/dict_tests/dictionary): everything between its
    ID and its repeat offsets, which are 1, 4, 8."""
    raw = open(os.path.join(HERE, "golden", "dict_tests", "dictionary"), "rb").read()
    end = raw.find(struct.pack("<3I", 1, 4, 8))
    return raw[8:end]


GOLDEN_TABLES = _golden_tables()


class Dict:
    """A dictionary: formatted (magic, ID, the golden tables, `reps`, content) or raw content (reps None: [1, 4, 8])."""

    def __init__(self, name, dict_id, content, reps=None):
        self.name, self.id, self.content = name, dict_id, bytes(content)
        self.formatted = reps is not None
        self.reps = tuple(reps) if reps is not None else (1, 4, 8)
        self.raw = (struct.pack("<II", 0xEC30A437, dict_id) + GOLDEN_TABLES + struct.pack("<3I", *self.reps) + self.content
                    if self.formatted else None)

    def __repr__(self):
        return self.name


# ---------------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------------
class Result:
    """out: the content produced (up to the failing sequence); err: None or (error leaf, stage); reaches: per sequence that
    reached past the buffer, (block, index in block, counter before it, from_dict, "full" | "straddle" | None); fail: (block,
    index, counter) of the failing sequence."""

    def __init__(self):
        self.out, self.err, self.reaches, self.fail = bytearray(), None, [], None

    @property
    def outcome(self):
        return ERROR if self.err else bytes(self.out)


def execute(blocks, dict_content=b"", reps=None, window_size=1 << 17, drains=None, rfc=False, cap=None):
    """The frame's content or its error.  reps: a formatted dictionary's repeat offsets (None: [1, 4, 8], as for a raw-content
    dictionary or none).  drains[i]: bytes read out after block i, as the reference's read does (only down to window_size while
    the frame is unfinished).  cap: the output capacity (TargetTooSmall, stage drain, at the first byte that does not fit)."""
    r = Result()
    out = r.out
    dl = len(dict_content)
    if rfc and reps is not None and any(v == 0 or v > dl for v in reps):
        r.err = ("dictionary", 0)
        return r
    h = list(reps if reps is not None else (1, 4, 8))
    counter = drained = 0

    def fits(n):
        return cap is None or len(out) + n <= cap

    for bi, b in enumerate(blocks):
        if b[0] in ("raw", "rle"):
            data = bytes(b[1]) if b[0] == "raw" else bytes([b[1]]) * b[2]
            if not fits(len(data)):
                r.err = ("ERR_TARGET_TOO_SMALL", STAGE_DRAIN)
                return r
            out += data                                    # extend_from_reader / extend_and_fill: counter untouched
        else:
            lits, seqs = b[1], b[2]
            li = 0
            for si, (ll, ml, ov) in enumerate(seqs):
                if ll > 0:
                    if li + ll > len(lits):
                        r.err = ("ERR_EXEC_NOT_ENOUGH_BYTES_FOR_SEQUENCE", STAGE_EXECUTE)
                        return r
                    if not fits(ll):
                        r.err = ("ERR_TARGET_TOO_SMALL", STAGE_DRAIN)
                        return r
                    out += lits[li:li + ll]
                    li += ll
                    counter += ll
                off = S.offset_history(ov, ll, h)
                if off == 0:
                    r.err = ("ERR_EXEC_ZERO_OFFSET", STAGE_EXECUTE)
                    return r
                if ml == 0:
                    continue
                if not fits(ml):
                    r.err = ("ERR_TARGET_TOO_SMALL", STAGE_DRAIN)
                    return r
                if rfc:
                    if off > len(out) + dl or off > window_size:
                        r.err = ("offset", 0)
                        return r
                    for _ in range(ml):                    # the history is the dictionary followed by the output
                        p = dl + len(out) - off
                        out.append(dict_content[p] if p < dl else out[p - dl])
                    continue
                buf_len = len(out) - drained
                if off <= buf_len:
                    for _ in range(ml):
                        out.append(out[-off])
                    counter += ml
                    continue
                # repeat_from_dict
                if counter > window_size:
                    r.err, r.fail = (TOO_BIG, STAGE_EXECUTE), (bi, si, counter)
                    r.reaches.append((bi, si, counter, None, None))
                    return r
                from_dict = off - buf_len
                if from_dict > dl:
                    r.err, r.fail = (NOT_IN_DICT, STAGE_EXECUTE), (bi, si, counter)
                    r.reaches.append((bi, si, counter, from_dict, None))
                    return r
                if from_dict < ml:
                    r.reaches.append((bi, si, counter, from_dict, "straddle"))
                    out += dict_content[dl - from_dict:]
                    counter += from_dict
                    rest, period = ml - from_dict, len(out) - drained   # repeat(buffer.len(), rest): from the buffer's start
                    for k in range(rest):
                        out.append(out[drained + k % period])
                    counter += rest
                else:
                    r.reaches.append((bi, si, counter, from_dict, "full"))
                    out += dict_content[dl - from_dict:dl - from_dict + ml]    # counter not advanced (:166-171)
            if li < len(lits):
                if not fits(len(lits) - li):
                    r.err = ("ERR_TARGET_TOO_SMALL", STAGE_DRAIN)
                    return r
                counter += len(lits) - li
                out += lits[li:]
        if drains is not None and not rfc and bi < len(drains):
            last = bi + 1 == len(blocks)
            assert last or drains[bi] <= max(0, len(out) - drained - window_size), "a read drains only down to the window"
            drained += drains[bi]
    return r


def window_of(window_log=17, window_desc=None, single_segment=False, content_size=None):
    """Window_Size of a frame header (RFC 8878 3.1.1.1.2; the content size for a Single_Segment frame)."""
    if single_segment:
        return content_size
    wd = (window_log - 10) << 3 if window_desc is None else window_desc
    base = 1 << (10 + (wd >> 3))
    return base + (base >> 3) * (wd & 7)


# ---------------------------------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------------------------------
def _content(seed, n):
    rng = random.Random(seed)
    return bytes(rng.randrange(256) for _ in range(n))


D_MAIN = Dict("main", 0x1234, _content(1, 300), (1, 4, 8))
D_ONE = Dict("one-byte", 0x1235, b"\x9c", (1, 1, 1))
D_LONG = Dict("long", 0x1236, _content(2, 4000), (1, 4, 8))
D_REPS = Dict("reps", 0x1237, _content(3, 300), (200, 150, 60))
D_REP1 = Dict("rep0=1", 0x1238, _content(4, 300), (1, 50, 60))
D_A = Dict("multi-a", 0x21, _content(5, 500), (77, 5, 300))
D_B = Dict("multi-b", 0x3344, _content(6, 700), (9, 650, 33))
D_R = Dict("multi-raw", 0x55, _content(7, 600))
REP_VALUES = {"0": 0, "2^30-1": (1 << 30) - 1, "2^30": 1 << 30, "2^31": 1 << 31, "2^32-1": (1 << 32) - 1}
D_WEIRD = {(name, slot): Dict(f"rep{slot}={name}", 0x4000 + 8 * i + slot, _content(8, 300),
                              tuple(v if k == slot else (30, 40, 50)[k] for k in range(3)))
           for i, (name, v) in enumerate(REP_VALUES.items()) for slot in range(3)}
DICTS = [D_MAIN, D_ONE, D_LONG, D_REPS, D_REP1, D_A, D_B, D_R] + list(D_WEIRD.values())


class Case:
    """One crafted frame.  dict: the dictionary the frame names by ID (None: no ID field); forced: the dictionary forced on the
    decoder instead (forced_dict / force_dict).  cap: the output capacity of the batch tier (None: the content's size).
    drains: a read schedule for the FrameDecoder tier.  handback: WHY_SEQ_CHECK when k_exec_cta must hand the frame back."""

    def __init__(self, group, name, blocks, dict=None, forced=None, window_log=17, window_desc=None, single_segment=False,
                 id_bytes=4, cap=None, drains=False, quirk=False, handback=None, libzstd=True):
        self.group, self.id = group, f"{group}-{name}"
        self.blocks, self.dict, self.forced, self.quirk, self.handback = blocks, dict, forced, quirk, handback
        self.window_log, self.window_desc, self.single_segment, self.id_bytes = window_log, window_desc, single_segment, id_bytes
        self.drains = drains
        self.use = forced if forced is not None else dict
        self.full = self.run()
        nominal = S.nominal_size(blocks)
        self.window = window_of(window_log, window_desc, single_segment, nominal)
        self.valid = self.full.err is None
        self.expected = self.full.outcome
        self.cap = (len(self.expected) if self.valid else max(1, nominal)) if cap is None else cap
        self.batch = self.run(cap=self.cap) if cap is not None else self.full
        # libzstd matches the frame's Dictionary_ID against the dictionary's, and raw content has none
        self.libzstd = libzstd and (self.dict is None or (self.use is self.dict and self.use.formatted))
        self._frame = None

    def run(self, rfc=False, drains=None, cap=None):
        d = self.use
        window = window_of(self.window_log, self.window_desc, self.single_segment, S.nominal_size(self.blocks))
        return execute(self.blocks, d.content if d else b"", d.reps if d is not None and d.formatted else None, window,
                       drains=drains, rfc=rfc, cap=cap)

    @property
    def frame(self):
        if self._frame is None:
            self._frame = S.frame(self.blocks, self.window_log, content_size=S.nominal_size(self.blocks), checksum=True, ov=True,
                                  plain=self.expected if self.valid else b"", dict_id=self.dict.id if self.dict else None,
                                  dict_id_bytes=self.id_bytes, single_segment=self.single_segment, window_desc=self.window_desc)[0]
        return self._frame

    def __repr__(self):
        return self.id


def skewed(rng, n):
    return S.skewed(rng, n)


def _lits(rng, seqs, tail=0):
    return skewed(rng, sum(q[0] for q in seqs) + tail)


def _ordinary(rng, n, pos, ml_hi=20, of_max=1 << 17):
    """n sequences with offsets inside the output so far (Offset_Value form, no repeat codes); pos = output before them."""
    seqs = []
    for _ in range(n):
        ll, ml = rng.randint(1, 3), rng.randint(3, ml_hi)
        seqs.append((ll, ml, rng.randint(1, min(pos + ll, of_max)) + 3))
        pos += ll + ml
    return seqs


def _new(of):
    return of + 3


def reach(rng):
    out = []
    d = D_MAIN
    dl = len(d.content)
    pre = _ordinary(rng, 10, 44)
    p0 = 44 + S._end(pre)

    def one(name, seq, dct=d, **kw):
        seqs = [(40, 4, _new(7))] + pre + [seq] + _ordinary(rng, 5, p0 + seq[0] + seq[1])
        out.append(Case("reach", name, [("cmp", _lits(rng, seqs, 3), seqs)], dict=dct, **kw))

    one("of=produced+dict_len", (6, 20, _new(p0 + 6 + dl)))
    one("of=produced+dict_len+1", (6, 20, _new(p0 + 6 + dl + 1)))
    one("from_dict=ml-full", (6, 40, _new(p0 + 6 + 40)))
    one("from_dict=ml-1-straddle-by-one", (6, 40, _new(p0 + 6 + 39)))
    one("from_dict=ml+1-full", (6, 40, _new(p0 + 6 + 41)))
    one("straddle-later-in-frame", (6, 100, _new(p0 + 6 + 20)))
    # the frame's first byte: buffer empty, 10 bytes from the dictionary, then 40 repeating the frame's first 10
    seqs = [(0, 50, _new(10))] + _ordinary(rng, 5, 50)
    out.append(Case("reach", "straddle-at-frame-start-periodic", [("cmp", _lits(rng, seqs, 2), seqs)], dict=d))
    one("one-byte-dict-straddle", (6, 5, _new(p0 + 6 + 1)), dct=D_ONE)
    one("one-byte-dict-of=produced+2", (6, 5, _new(p0 + 6 + 2)), dct=D_ONE)
    # the drain schedule with a dictionary: RLE blocks (not counted) then a straddle after a read, whose second part starts at
    # the retained buffer's first byte
    blocks = [("rle", 0x5A, 3000), ("raw", bytes(range(256)) * 4), ("cmp", skewed(rng, 4), [(2, 50, _new(2 + 1024 + 10)), (2, 6, _new(40))])]
    out.append(Case("reach", "straddle-after-read-drained", blocks, dict=D_MAIN, window_log=10, quirk=True, drains=True))
    # the same over 5 MiB: 128 KiB Raw blocks (not counted), each followed by a Compressed block whose straddle, after the reads,
    # takes its second part from the retained buffer's first byte.  Read block by block, a decoder that keeps the frame in a
    # growing window buffer and drops the drained bytes when it grows has moved that buffer several times before the later
    # straddles.
    W = 1 << 16
    blocks = []
    for k in range(40):
        blocks.append(("raw", rng.randbytes(S.BLOCK_MAX)))
        blocks.append(("cmp", skewed(rng, 2), [(2, 60, _new(W + 2 + 10 + k % 7))]))
    out.append(Case("reach", "straddle-after-read-window-buffer-growth-drained", blocks, dict=D_MAIN, window_log=16, quirk=True,
                    drains=True))
    # a dictionary longer than the window: reachable up to its first byte while the counter is within the window
    seqs = [(30, 20, _new(30 + 3000)), (2, 30, _new(32 + 20 + 3900))]
    out.append(Case("reach", "dict-longer-than-window", [("cmp", _lits(rng, seqs, 2), seqs)], dict=D_LONG, window_log=10, quirk=True))
    return out


def counter(rng):
    """The counter rule at a 1 KiB window and at a window with a mantissa: counted bytes before the reach of exactly W and W + 1."""
    out = []
    d = D_MAIN
    for wname, wlog, wdesc in (("w1KiB", 10, None), ("w1408-mantissa3", 10, 3)):
        W = window_of(wlog, wdesc)
        for extra in (0, 1):
            ok = extra == 0
            tag = "W" if ok else "W+1"
            probe = lambda p: ("cmp", skewed(rng, 2), [(0, 12, _new(p + 20))])         # from_dict = 20, a full copy
            kw = dict(dict=d, window_log=wlog, window_desc=wdesc, quirk=ok)
            # through literals
            blocks = [("cmp", skewed(rng, W + extra), [])]
            out.append(Case("counter", f"{wname}-literals-counter={tag}", blocks + [probe(W + extra)], **kw))
            # through in-buffer matches
            n = W + extra
            blocks = [("cmp", skewed(rng, 10), [(10, n - 10, _new(3))])]
            out.append(Case("counter", f"{wname}-matches-counter={tag}", blocks + [probe(n)], **kw))
            # through a straddle: 20 bytes from the dictionary and the rest repeating them
            blocks = [("cmp", b"", [(0, n, _new(20))])]
            out.append(Case("counter", f"{wname}-straddle-counter={tag}", blocks + [probe(n)], **kw))
    # 100 KiB of Raw / RLE blocks first: not counted, the dictionary is still reachable
    raw = bytes(rng.randrange(256) for _ in range(S.BLOCK_MAX))
    rle_blocks = [("rle", 0x61, 100 * 1024)]
    raw_blocks = [("raw", raw[:60 * 1024]), ("raw", raw[:40 * 1024])]
    for name, blocks in (("rle-100KiB", rle_blocks), ("raw-100KiB", raw_blocks)):
        p = S.nominal_size(blocks)
        out.append(Case("counter", f"{name}-then-reach", blocks + [("cmp", skewed(rng, 8), [(4, 30, _new(p + 4 + 200)), (4, 9, _new(100))])],
                        dict=d, window_log=10, quirk=True))
    # copies wholly from the dictionary totalling 1500 > W bytes: not counted, the dictionary is still reachable after them
    seqs, p = [], 0
    for k in range(15):
        seqs.append((2, 100, _new(p + 2 + 100 + 3 * k)))
        p += 102
    seqs.append((2, 10, _new(p + 2 + 250)))
    out.append(Case("counter", "full-copies-1500-uncounted", [("cmp", _lits(rng, seqs, 1), seqs)], dict=D_LONG, window_log=10, quirk=True))
    # Single_Segment: the window is the content size
    seqs = [(50, 30, _new(50 + 60)), (5, 40, _new(85))]
    out.append(Case("counter", "single-segment-reach-inside-window", [("cmp", _lits(rng, seqs, 7), seqs)], dict=d, single_segment=True))
    seqs = [(50, 30, _new(50 + 280)), (5, 40, _new(5 + 80))]
    out.append(Case("counter", "single-segment-reach-beyond-content-size", [("cmp", _lits(rng, seqs, 7), seqs)], dict=d,
                    single_segment=True, quirk=True))
    return out


def reps(rng):
    """A dictionary's repeat offsets as the history of the frame's first Compressed block, in the first block and after Raw,
    RLE and zero-sequence Compressed blocks."""
    out = []
    d = D_REPS                         # [200, 150, 60], content 300: every one reaches into the content from the frame's start
    for ov in (1, 2, 3):
        for ll in (0, 5):
            seqs = [(ll, 12, ov), (2, 6, 1), (0, 5, 2)]
            out.append(Case("reps", f"ov{ov}-ll{ll}-into-content", [("cmp", _lits(rng, seqs, 3), seqs)], dict=d))
    out.append(Case("reps", "rep0=1-ov3-ll0-offset0", [("cmp", skewed(rng, 1), [(0, 4, 3)])], dict=D_REP1))
    seps = {"first": [], "after-raw": [("raw", b"qrs" * 5)], "after-rle": [("rle", 0x42, 300)],
            "after-cmp0seq": [("cmp", skewed(rng, 20), [])]}
    for (name, slot), dd in D_WEIRD.items():
        # ll > 0: codes 1-3 are slots 0-2; ll = 0: codes 1, 2 are slots 1, 2 and code 3 is slot 0 minus one
        for sep, mid in seps.items():
            seqs = [(4, 6, slot + 1), (3, 5, _new(2))]
            blocks = mid + [("cmp", _lits(rng, seqs, 2), seqs)]
            out.append(Case("reps", f"rep{slot}={name}-ll4-{sep}", blocks, dict=dd))
        if slot == 0:
            seqs = [(0, 6, 3), (3, 5, _new(2))]
            out.append(Case("reps", f"rep0={name}-ov3-ll0-minus-one", [("cmp", _lits(rng, seqs, 2), seqs)], dict=dd))
            # never used: the reference accepts the dictionary (the format does not), and the value moves through the history
            seqs = [(4, 6, 2), (3, 5, _new(2)), (2, 4, 1)]
            out.append(Case("reps", f"rep0={name}-unused", [("cmp", _lits(rng, seqs, 2), seqs)], dict=dd, quirk=True))
        elif slot in (1, 2):
            seqs = [(0, 6, slot), (3, 5, _new(2))]
            out.append(Case("reps", f"rep{slot}={name}-ll0-code{slot}", [("cmp", _lits(rng, seqs, 2), seqs)], dict=dd))
    return out


def batch(rng):
    """A dictionary-reaching sequence at chosen indices of a block of ordinary sequences; the exact-path replay of k_fse."""
    out = []
    d = D_MAIN
    for idx in (0, 63, 64, 65, 127, 128):
        seqs = ([(8, 5, _new(3))] + _ordinary(rng, idx - 1, 13)) if idx else []
        pos = S._end(seqs)
        seqs.append((2, 30, _new(pos + 2 + 100)))          # 100 bytes into the dictionary: a full copy
        seqs += _ordinary(rng, 200 - idx - 1, pos + 32)
        assert len(seqs) == 200
        out.append(Case("batch", f"reach-at-seq{idx}", [("cmp", _lits(rng, seqs, 4), seqs)], dict=d))
    for ofcode in (8, 9):
        xbits = 15 + 15 + ofcode
        pre = [(16, 5, _new(7))] + _ordinary(rng, 9, 21)
        pos = S._end(pre)
        pre += [(3, 40, _new(pos + 3 + 60))]                  # a full copy: 40 of the dictionary's last 60 bytes
        pre += [(3, 80, _new(S._end(pre) + 3 + 25))]          # a straddle: 25 from the dictionary, 55 from the frame's start
        pre += _ordinary(rng, 300, S._end(pre), ml_hi=10)
        pos = S._end(pre)
        wide = (32768 + rng.randrange(8000), 32771 + rng.randrange(8000), 1 << ofcode)
        seqs = pre + [wide] + _ordinary(rng, 40, pos + wide[0] + wide[1])
        name = f"reach-then-xbits{xbits}" + ("-replay" if xbits > FSE_FAST_XBITS else "-no-replay")
        c = Case("batch", name, [("cmp", _lits(rng, seqs, 3), seqs)], dict=d)
        c.xbits = xbits
        out.append(c)
    return out


def nodict(rng):
    """No dictionary: offsets past the window but inside the produced bytes; the NotEnoughBytesInDictionary / OffsetTooBig flip."""
    out = []
    W = 1024
    # 3000 produced, an offset of 2000 > W: accepted while nothing is drained; after a read keeps only W bytes it is not
    first = [(40, 4, _new(9))] + _ordinary(rng, 250, 44, of_max=W)
    assert S._end(first) > 2000
    seqs2 = [(5, 20, _new(2000)), (0, 8, _new(1500))]
    blocks = [("cmp", _lits(rng, first, 5), first), ("cmp", _lits(rng, seqs2, 3), seqs2)]
    out.append(Case("nodict", "of-past-window-inside-produced", blocks, window_log=10, quirk=True))
    out.append(Case("nodict", "of-past-window-inside-produced-drained", blocks, window_log=10, quirk=True, drains=True))
    raw = ("raw", bytes(rng.randrange(256) for _ in range(3000)))
    for extra, leaf in ((0, "W"), (1, "W+1")):
        for pre_name, pre in (("", []), ("raw3000-", [raw])):
            # block A counts W + extra - 13 bytes, block B 13 more before the offset one past the produced bytes
            p = S.nominal_size(pre)
            n = W + extra - 13
            blocks = pre + [("cmp", skewed(rng, 200), [(100, n - 200, _new(37))]),
                            ("cmp", skewed(rng, 6), [(3, 7, _new(12)), (3, 5, _new(p + n + 13 + 1))])]
            out.append(Case("nodict", f"{pre_name}counter={leaf}", blocks, window_log=10, handback=WHY_SEQ_CHECK))
    return out


def multi(rng):
    out = []
    for dd in (D_A, D_B, D_R):
        for nb in ((1, 2, 4) if dd.id < 256 else (2, 4)):
            dl = len(dd.content)
            seqs = [(7, 15, _new(7 + dl - 3)), (2, 9, 1), (0, 11, 2), (4, 6, _new(20))]
            out.append(Case("multi", f"{dd.name}-id{nb}B", [("cmp", _lits(rng, seqs, 2), seqs)], dict=dd, id_bytes=nb))
    seqs = [(7, 15, _new(7 + 400)), (2, 9, 1), (0, 11, 2)]
    out.append(Case("multi", "forced-b-over-id-a", [("cmp", _lits(rng, seqs, 2), seqs)], dict=D_A, forced=D_B, id_bytes=1))
    out.append(Case("multi", "forced-raw-no-id", [("cmp", _lits(rng, seqs, 2), seqs)], forced=D_R))
    return out


def cap(rng):
    out = []
    # 24 bytes, then 6 literals and a 50-byte match starting at 30 that ends past the capacity
    seqs = [(20, 4, _new(5)), (6, 50, _new(24 + 6 + 100))]          # 50 of the dictionary's last 100 bytes
    out.append(Case("cap", "inside-full-copy", [("cmp", _lits(rng, seqs, 3), seqs)], dict=D_MAIN, cap=24 + 6 + 20))
    seqs = [(20, 4, _new(5)), (6, 50, _new(24 + 6 + 10))]           # 10 from the dictionary, 40 from the frame's start
    out.append(Case("cap", "inside-straddle-second-part", [("cmp", _lits(rng, seqs, 3), seqs)], dict=D_MAIN, cap=24 + 6 + 25))
    return out


GROUPS = {"reach": reach, "counter": counter, "reps": reps, "batch": batch, "nodict": nodict, "multi": multi, "cap": cap}


def cases(group=None):
    """The crafted cases (all groups, or one), built from fixed seeds."""
    out = []
    for i, (g, fn) in enumerate(GROUPS.items()):
        if group is None or g == group:
            out += fn(random.Random(0xD1C0 + i))
    return out


def oracle_decoder(oracle):
    """An oracle FrameDecoder with every dictionary added."""
    d = oracle.FrameDecoder()
    for dd in DICTS:
        if dd.formatted:
            d.add_dict(dd.raw)
        else:
            d.add_raw_content_dict(dd.id, dd.content)
    return d


def oracle_decode(oracle, c):
    """Decodes case `c` with the oracle (decode_blocks(All) + collect); checks that its trace holds exactly the requested
    sequences up to where it stopped.  Returns (content, None) or (None, (error leaf, stage))."""
    d = oracle_decoder(oracle)
    d.trace_enable()
    try:
        r = d.reset(c.frame)
        if c.forced is not None:
            d.force_dict(c.forced.id)
        d.decode_blocks(r, oracle.ALL)
        res = (d.collect(), None)
    except oracle.OracleError as e:
        res = (None, (oracle.error_names()[e.code].replace("ZO_", ""), e.stage))
    _, _, seqs = d.trace()
    want = [q for b in c.blocks if b[0] == "cmp" for q in b[2]]
    got = [tuple(int(x) for x in s[:3]) for s in seqs]
    assert got == want[:len(got)], "the oracle decoded other sequences than the ones requested"
    if res[1] is None:
        assert len(got) == len(want)
    return res


def oracle_drained(oracle, c):
    """The drain schedule on the oracle: decode_blocks(UptoBlocks, 1) then read everything it can collect, per block.  Returns
    (content, error or None, bytes read after each block, [(can_collect after the block, bytes read)])."""
    d = oracle_decoder(oracle)
    r = d.reset(c.frame)
    if c.forced is not None:
        d.force_dict(c.forced.id)
    out, drains, steps = bytearray(), [], []
    try:
        while not d.is_finished():
            d.decode_blocks(r, oracle.UPTO_BLOCKS, 1)
            cc = d.can_collect()
            got = d.read(cc)
            steps.append((cc, len(got)))
            drains.append(len(got))
            out += got
    except oracle.OracleError as e:
        return bytes(out), (oracle.error_names()[e.code].replace("ZO_", ""), e.stage), drains, steps
    out += d.collect()
    return bytes(out), None, drains, steps
