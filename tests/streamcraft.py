"""Crafted frames put across the cuts of the stream decoder (decode_all_stream, tier 1d), shared by the CPU and GPU tests.

decode_all_stream is the one decode path that stops a frame at one submission and finishes it in a later one.  At each cut it
carries the frame's tables (the planner's copy into the carry slot, or a re-pointed table), its offset history and
total_output_counter (k_carry), its last T = min(produced, max(window, 32)) bytes (k_carry's shifted 16-byte copy), its
placement (k_place_resume) and its checksum accumulators (k_xxh64_stream, which reads the bytes after the last whole 32-byte
stripe back from the tail).  This module puts every crafted decoder case (tests/seqcraft.py, entcraft.py, hufring.py,
dictcraft.py) across cuts, adds families built so that each of those carried pieces is used right after a cut, and states how
a stream of cases is laid out and what each cut carries -- computed from the cut model (tests/streamcut.py) and the blocks'
decoded sizes, with no GPU.

Every case is one frame in the blocks form of seqcraft with Offset_Value sequences: ("raw", bytes), ("rle", byte, count),
("cmp", literals, [(ll, ml, offset_value), ...]).  A stream at chunk size C is, per case, a skippable frame, the case's lead
frame (optional) and the case's frame.  Below the default chunk the skippable frame is C bytes long, so it always ends the
submission in front of it and every case starts a fresh submission: where the cuts fall in a case depends only on the case and
C.  A lead frame of r bytes then sits in the same submission as the case's first blocks and moves where the case is placed."""
import random

import dictcraft as D
import entcraft as E
import hufring as H
import seqcraft as S
import streamcut
from test_decode_all_chain import skippable

ERROR = S.ERROR
BLOCK_MAX = S.BLOCK_MAX
DEFAULT = 64 << 20
# A Compressed block counts min(128 KiB, window) against the output bound 4 C.  4096: one block per submission, so every block
# boundary is a cut.  32768: two blocks, one Compressed block of a 128 KiB window.  65536: four blocks, two such Compressed
# blocks.  196608: twelve blocks, six of them.  The default cuts none of these streams.
CHUNKS = (4096, 32768, 65536, 196608, DEFAULT)
TABLES = ("huf", "ll", "of", "ml")


def keep(window):
    """Bytes a continuing frame carries at most: max(window, 32)."""
    return max(window, 32)


# ---------------------------------------------------------------------------------------------------------------------------
# one case
# ---------------------------------------------------------------------------------------------------------------------------
class Case:
    """One frame.  kind: the builder ("seq", "ent", "dict", or "seqframe" for seqcraft.frame with its header options), src its
    case object.  dicts: the dictionary set the frame needs ("dictcraft": tests/dictcraft.py's, "entcraft": formatted
    dictionaries built with entcraft.dictionary, None); forced: the dictcraft Dict forced on the decoder.  lead: the bytes of the
    lead frame in front of it, lead_plain what that decodes to.  reps: the offset history the frame starts from."""

    def __init__(self, group, name, kind, src, frame, blocks, expected, reps=(1, 4, 8), dicts=None, dict_raw=None, forced=None,
                 lead=b"", lead_plain=b"", libzstd=True, tables0=None):
        self.group, self.id, self.kind, self.src = group, name if name.startswith(group + "-") else f"{group}-{name}", kind, src
        self.frame, self.blocks, self.expected = frame, blocks, expected
        self.valid = expected is not ERROR
        self.reps, self.dicts, self.dict_raw, self.forced = tuple(reps), dicts, dict_raw, forced
        self.lead, self.lead_plain, self.libzstd = lead, lead_plain, libzstd
        err, self.hlen, self.window, self.checksum = frame_header(frame)
        assert err is None, (self.id, err)
        # the same frame with a Dictionary_ID of 0 (no dictionary), which the cut model reads as the decoder cuts the frame
        d = frame[4]
        did, at = [0, 1, 2, 4][d & 3], 6 - ((d >> 5) & 1)
        self.cut_frame = bytes(frame[:at]) + bytes(did) + bytes(frame[at + did:])
        self.sizes = [block_size(b) for b in blocks]
        # the tables the frame starts with: a formatted dictionary's (none of these frames starts otherwise)
        self.tables0 = tables0

    def __repr__(self):
        return self.id


def frame_header(frame):
    """streamcut.frame_header's (error, header length, window, checksum flag) of a zstd frame, read past its Dictionary_ID."""
    d = frame[4]
    did, at = [0, 1, 2, 4][d & 3], 6 - ((d >> 5) & 1)
    err, hl, window, checksum, _ = streamcut.frame_header(bytes(frame[:4]) + bytes([d & ~3]) + bytes(frame[5:at]) + bytes(frame[at + did:18 + did]))
    return err, hl + did, window, checksum


def block_size(b):
    """Bytes the block decodes to when every sequence executes."""
    if b[0] == "raw":
        return len(b[1])
    if b[0] == "rle":
        return b[2]
    return len(b[1]) + sum(q[1] for q in b[2])


def offsets(blocks, reps=(1, 4, 8)):
    """The actual offset of every sequence, in order (RFC 8878 3.1.2.5; Raw and RLE blocks leave the history alone)."""
    h, out = list(reps), []
    for b in blocks:
        if b[0] == "cmp":
            for ll, ml, ov in b[2]:
                out.append(S.offset_history(ov, ll, h))
    return out


def deviation(c):
    """Why case `c` lies outside what tier 1d promises to decode as decode_all_batch does (DESIGN.md 4.9, "History"), or None:
    a sequence's offset exceeds the window (the tail holds max(window, 32) bytes), or a Compressed block decodes to more than its
    min(128 KiB, window) bound in the submission's output room."""
    if any(o > c.window for o in offsets(c.blocks, c.reps)):
        return "offset-past-window"
    if any(b[0] == "cmp" and n > min(BLOCK_MAX, c.window) for b, n in zip(c.blocks, c.sizes)):
        return "block-output-limit"
    return None


def _ov_blocks(blocks, ov):
    return [b if b[0] != "cmp" or ov else ("cmp", b[1], [(ll, ml, of + 3) for ll, ml, of in b[2]]) for b in blocks]


def from_seq(c, group=None):
    return Case(group or "seqcraft", c.id, "seq", c, c.frame, _ov_blocks(c.blocks, c.ov), c.expected)


def from_ent(c, group=None, **kw):
    raw = c.dict_raw
    return Case(group or ("hufring" if c.group == "huf-ring" else "entcraft"), c.id, "ent", c, c.frame, E.plain_blocks(c.blocks),
                c.expected, dicts="entcraft" if raw is not None else None, dict_raw=raw, libzstd=c.libzstd,
                tables0="dictionary" if raw is not None else None, **kw)


def from_dict(c):
    d = c.use
    return Case("dictcraft", c.id, "dict", c, c.frame, c.blocks, c.expected, reps=d.reps if d is not None and d.formatted else (1, 4, 8),
                dicts="dictcraft", forced=c.forced, libzstd=c.libzstd, tables0="dictionary" if d is not None and d.formatted else None)


def crafted():
    """Every case of seqcraft.cases(), entcraft.cases(), hufring.cases() and dictcraft.cases(), with its checksum wherever the
    builder writes one (every valid case)."""
    return ([from_seq(c) for c in S.cases()] + [from_ent(c) for c in E.cases()] + [from_ent(c) for c in H.cases()] +
            [from_dict(c) for c in D.cases()])


# ---------------------------------------------------------------------------------------------------------------------------
# the stream-edge families
# ---------------------------------------------------------------------------------------------------------------------------
def lead_frame(plain):
    """A frame of one Raw block holding `plain`, with its checksum."""
    return S.frame([("raw", plain)], 20, content_size=None, checksum=True)[0]


def _lead(n):
    plain = bytes((i * 37 + 11) & 0xFF for i in range(n))
    return lead_frame(plain), plain


def _ent(group, name, blocks, window_log=17, lead=None, **kw):
    c = E.Case(group, name, blocks, window_log=window_log, **kw)
    lf, lp = _lead(lead) if lead is not None else (b"", b"")
    return from_ent(c, group=group, lead=lf, lead_plain=lp)


def _seqframe(group, name, blocks, window_log=17, lead=None, libzstd=True, **kw):
    frame = S.frame(blocks, window_log, checksum=True, ov=True, **kw)[0]
    lf, lp = _lead(lead) if lead is not None else (b"", b"")
    return Case(group, name, "seqframe", None, frame, blocks, S.execute(blocks, ov=True), lead=lf, lead_plain=lp, libzstd=libzstd)


def _rawlits(seqs, rng, tail=3):
    """A Compressed block of Raw literals and predefined tables holding `seqs` (any codes the predefined tables have)."""
    return E.Blk(bytes(rng.randrange(256) for _ in range(sum(q[0] for q in seqs) + tail)), "raw", seqs=seqs, modes=[("pre",)] * 3)


def _ordinary(rng, n, pos, ml_hi=20, of_max=BLOCK_MAX):
    """n sequences with new offsets inside the output so far (Offset_Value form); pos = output before them."""
    seqs = []
    for _ in range(n):
        ll, ml = rng.randint(1, 4), rng.randint(3, ml_hi)
        seqs.append((ll, ml, rng.randint(1, min(pos + ll, of_max)) + 3))
        pos += ll + ml
    return seqs


def _nominal(blocks):
    return S.nominal_size(E.plain_blocks(blocks))


def carry_tables(rng):
    """Each table kind as the block right after a cut (at 4096 every block is its own submission): Treeless literals with 1 and
    4 streams, Repeat of FSE, RLE and predefined tables (all three, and one kind at a time), a cut where LL is new and OF / ML
    repeat (the carry slot then holds a copied table beside kept ones), Treeless + Repeat over four cuts in a row, and the tables
    of a formatted dictionary taken by Repeat after a cut."""
    out = []
    g = "carry-tables"
    h = E.Huf(E.lengths_for(rng, range(40), 8))
    L = lambda n, hh=h: E.literals(rng, hh.lengths, n)
    for streams in (1, 4):
        out.append(_ent(g, f"treeless-{streams}stream", [E.Blk(L(600), huf=h), E.Blk(L(500), "treeless", streams=streams)]))
    fse = lambda log: ("fse", log, E.rand_norm(rng, 20, log, neg=1, keep=(2, 3, 4)))
    defs = {"fse": [fse(6), fse(5), fse(7)], "rle": [("rle", 4), ("rle", 6), ("rle", 9)], "pre": [("pre",)] * 3}
    for d, modes in defs.items():
        b0 = E.seq_block(rng, modes, 50)
        b1 = E.seq_block(rng, [("rep",)] * 3, 70, pos=64 + _nominal([b0]), codes=E.codes_of(modes))
        out.append(_ent(g, f"repeat-all-of-{d}", [E.prefix(rng), b0, b1]))
    for k, kind in enumerate(E.KINDS):
        modes = [("pre",)] * 3
        modes[k] = ("rep",)
        b0 = E.seq_block(rng, defs["fse"], 50)
        b1 = E.seq_block(rng, modes, 60, pos=64 + _nominal([b0]), codes=E.codes_of(modes, E.codes_of(defs["fse"])))
        out.append(_ent(g, f"repeat-{kind}-of-fse", [E.prefix(rng), b0, b1]))
    b0 = E.seq_block(rng, defs["fse"], 50)
    mixed = [fse(6), ("rep",), ("rep",)]
    c1 = E.codes_of(mixed, E.codes_of(defs["fse"]))
    b1 = E.seq_block(rng, mixed, 50, pos=64 + _nominal([b0]), codes=c1)
    b2 = E.seq_block(rng, [("rep",)] * 3, 50, pos=64 + _nominal([b0, b1]), codes=c1)
    out.append(_ent(g, "ll-new-of-ml-kept", [E.prefix(rng), b0, b1, b2]))
    # a Huffman table and FSE tables built once, then Treeless + Repeat in four blocks in a row (Raw blocks between two of them)
    b0 = E.seq_block(rng, defs["fse"], 40, lit_mode="huf", huf=h)
    blocks, pos = [E.prefix(rng), b0], 64 + _nominal([b0])
    for i in range(4):
        if i == 2:
            blocks.append(("raw", bytes(rng.randrange(256) for _ in range(50))))
            pos += 50
        b = E.seq_block(rng, [("rep",)] * 3, 30 + 10 * i, pos=pos, lit_mode="treeless", huf=h, codes=E.codes_of(defs["fse"]))
        b.streams = 1 + 3 * (i & 1)
        blocks.append(b)
        pos += _nominal([b])
    out.append(_ent(g, "treeless-repeat-over-4-cuts", blocks))
    # a formatted dictionary's tables, taken by Treeless and Repeat after a cut: its first Compressed block is the second block
    dh = E.fse_weights(rng, E.lengths_for(rng, range(256), 11), 6, 1)
    of, ml, ll = (7, E.rand_norm(rng, 20, 7, neg=2, keep=(2, 3, 4, 5))), (7, E.rand_norm(rng, 30, 7, neg=2, keep=(0, 1, 2))), \
        (6, E.rand_norm(rng, 22, 6, neg=1, keep=(0, 1, 2)))
    raw, st = E.dictionary(DICT_ID, dh, of, ml, ll, (1, 4, 8), bytes(rng.randrange(256) for _ in range(200)))
    codes = {"ll": [s for s in range(22) if ll[1][s]], "of": [s for s in range(2, 7) if of[1][s]], "ml": [s for s in range(30) if ml[1][s]]}
    blocks, pos = [E.prefix(rng)], 64
    for n in (60, 40, 30):
        b = E.seq_block(rng, [("rep",)] * 3, n, pos=pos, lit_mode="treeless", huf=dh, codes=codes)
        blocks.append(b)
        pos += _nominal([b])
    c = E.Case(g, "dictionary-tables-by-repeat", blocks, dict_raw=raw, dict_id=DICT_ID, dict_state=st)
    out.append(from_ent(c, group=g))
    return out


DICT_ID = 0x5C0D      # the formatted dictionary of carry-tables (entcraft's own dictionary case uses 0x1234)


def carry_history(rng):
    """The offset history across a cut: repeat codes 1-3 with LL > 0 and the LL = 0 shifts as the first sequences of the block
    after a cut, rep0 - 1 down to 1 and saturating to 0 (an error), and a block on k_fse's exact path (LL code 34, ML code 51
    and OF code 9: 39 extra bits) right after one cut and right before the next, followed by repeat codes."""
    out = []
    g = "carry-history"
    head = [(20, 4, 13 + 3), (5, 4, 9 + 3), (5, 4, 17 + 3)]            # history [17, 9, 13]
    for ov in (1, 2, 3):
        for ll in (0, 6):
            tail = [(ll, 5, ov), (0, 4, 1), (2, 6, 3), (0, 3, 2), (1, 7, 50 + 3), (0, 4, 3)]
            out.append(_ent(g, f"ov{ov}-ll{ll}-first-after-cut", [_rawlits(head, rng), _rawlits(tail, rng)]))
    out.append(_ent(g, "ov3-ll0-rep0=2-after-cut", [_rawlits([(10, 4, 2 + 3)], rng), _rawlits([(0, 4, 3), (0, 5, 1), (2, 3, 3)], rng)]))
    out.append(_ent(g, "ov3-ll0-rep0=1-offset0-after-cut", [_rawlits([(10, 4, 1 + 3)], rng), _rawlits([(0, 4, 3), (3, 5, 2)], rng)]))
    for name, lead_blocks in (("exact-path-between-cuts", 1), ("exact-path-after-raw", 2)):
        pre = [("raw", bytes(rng.randrange(256) for _ in range(2000)))] * lead_blocks
        pos = 2000 * lead_blocks
        s0 = [(16, 5, 7 + 3)] + _ordinary(rng, 60, pos + 21, of_max=pos)
        b0 = _rawlits(s0, rng)
        pos += _nominal([b0])
        s1 = [(2, 6, 2)] + _ordinary(rng, 30, pos + 8, of_max=pos)
        p1 = pos + S._end(s1)
        wide = (32768 + rng.randrange(8000), 32771 + rng.randrange(8000), 512 + rng.randrange(512))
        s1 += [wide] + _ordinary(rng, 20, p1 + wide[0] + wide[1], of_max=5000) + [(4, 9, 1), (0, 7, 2)]
        b1 = _rawlits(s1, rng)
        pos += _nominal([b1])
        s2 = [(3, 8, 1), (0, 6, 1), (2, 5, 2), (0, 4, 3)] + _ordinary(rng, 30, pos + 23, of_max=5000)
        blocks = pre + [b0, b1, _rawlits(s2, rng)]
        out.append(_ent(g, name, blocks))
    return out


def tail_reach(rng):
    """Matches right after a cut whose source lies in the carried tail: its first byte (offset = window, with produced >=
    window; or the frame's first byte while produced < window), its last byte, a match straddling the tail and the new output,
    and an overlapping match that starts in the tail.  Three Raw blocks come first: at 4096 the cut in front of the reach follows
    a submission where the frame was resumed; at 65536 (four blocks) one where it follows its lead frame."""
    out = []
    g = "tail-reach"
    for wlog, sizes in ((10, (700, 800, 300)), (17, (700, 800, 300))):
        W = 1 << wlog
        P = sum(sizes)
        T = min(P, keep(W))
        firsts = {"first-byte": [(0, 20, T + 3)] if T == W else [(5, 20, T + 5 + 3)],
                  "last-byte-ll0": [(0, 20, 1 + 3)], "last-byte-ll5": [(5, 20, 6 + 3)],
                  "straddle": [(5, 30, 15 + 3)], "overlap-in-tail": [(0, 40, 5 + 3)]}
        for name, first in firsts.items():
            for lead in (None, 100):
                blocks = [("raw", bytes(rng.randrange(256) for _ in range(n))) for n in sizes]
                s = first + _ordinary(rng, 8, P + S._end(first), of_max=min(W, 500))
                blocks.append(_rawlits(s, rng))
                blocks.append(_rawlits([(2, 9, 1), (1, 5, 40 + 3)], rng))
                out.append(_ent(g, f"w{W}-{name}" + ("-after-lead" if lead else ""), blocks, window_log=wlog, lead=lead))
    return out


def alignment(rng):
    """Where the tail starts and how much of it the checksum reads again.  residue: the tail's source address (out_off + produced
    - T) takes every residue mod 16, set by a lead frame of r bytes (at 65536, with the frame's first three blocks in the lead's
    submission) and by a Raw block of 48 + r bytes (at 4096, the frame resumed).  stripe: the frame's bytes before the cut take
    every value mod 32, with T = the window (1 KiB) and with T = produced (128 KiB window).  small: fewer than 32 bytes before
    the cut (T = produced, no stripe yet).  Single_Segment frames of fewer than 32 bytes and of 1000 bytes (a window that is not a
    multiple of 16), window 1 KiB frames with T = window far below produced, and zero-byte Raw and Compressed blocks as the last
    block before a cut."""
    out = []
    reach = lambda P, W: _rawlits([(0, 20, min(P, W) + 3), (2, 9, 1)] + _ordinary(rng, 5, P + 31, of_max=min(P, W, 500)), rng)
    for r in range(16):
        blocks = [("raw", bytes(rng.randrange(256) for _ in range(n))) for n in (1200, 56, 16)] + [reach(1272, 1024)]
        out.append(_ent("align-residue", f"lead{r}", blocks, window_log=10, lead=r))
        blocks = [("raw", bytes(rng.randrange(256) for _ in range(n))) for n in (1200, 48 + r)] + [reach(1248 + r, 1024)]
        out.append(_ent("align-residue", f"raw{48 + r}", blocks, window_log=10))
    for u in range(32):
        for wlog, first in ((10, 1100 + u), (17, 64 + u)):
            blocks = [("raw", bytes(rng.randrange(256) for _ in range(first))), reach(first, 1 << wlog),
                      ("raw", bytes(rng.randrange(256) for _ in range(7 + u))), _rawlits([(1, 8, 2), (2, 6, 30 + 3)], rng)]
            out.append(_ent("align-stripe", f"w{1 << wlog}-first{first}", blocks, window_log=wlog))
    for k in (1, 2, 15, 16, 17, 31):
        blocks = [("raw", bytes(rng.randrange(256) for _ in range(k))),
                  _rawlits([(2, 5, k + 2 + 3), (0, 4, 1 + 3)], rng), _rawlits([(1, 6, 3 + 3)], rng)]
        out.append(_ent("align-small", f"produced{k}", blocks))
    g = "align-window"
    for n in (12, 21, 31):
        a, b = (n - 10) // 2, (n - 10) - (n - 10) // 2
        blocks = [("raw", bytes(rng.randrange(256) for _ in range(a))), ("raw", bytes(rng.randrange(256) for _ in range(b))),
                  ("cmp", bytes(rng.randrange(256) for _ in range(2)), [(2, 8, a + b + 2 + 3)])]
        out.append(_seqframe(g, f"single-segment-content{n}", blocks, single_segment=True))
    blocks = [("raw", bytes(rng.randrange(256) for _ in range(600))), ("raw", bytes(rng.randrange(256) for _ in range(301))),
              ("cmp", bytes(rng.randrange(256) for _ in range(7)), [(3, 40, 901 + 3 + 3), (4, 30, 37 + 3), (0, 22, 5 + 3)])]
    out.append(_seqframe(g, "single-segment-window1000", blocks, single_segment=True))
    blocks = [("raw", bytes(rng.randrange(256) for _ in range(1024))) for _ in range(6)]
    blocks += [reach(6144, 1024), ("rle", 0x61, 1024), reach(7300, 1024)]
    out.append(_ent(g, "w1024-T=window-produced6144", blocks, window_log=10))
    blocks = [("raw", bytes(rng.randrange(256) for _ in range(300))), ("raw", b""), reach(300, BLOCK_MAX)]
    out.append(_ent(g, "zero-byte-raw-before-cut", blocks))
    blocks = [("raw", bytes(rng.randrange(256) for _ in range(300))), E.Blk(b"", "raw"), reach(300, BLOCK_MAX)]
    out.append(_ent(g, "zero-byte-compressed-before-cut", blocks))
    blocks = [("raw", bytes(rng.randrange(256) for _ in range(300))), ("raw", b""), E.Blk(b"", "raw"), ("raw", b""), reach(300, BLOCK_MAX)]
    out.append(_ent(g, "zero-byte-blocks-over-3-cuts", blocks))
    return out


def cta_shape(rng):
    """A resumed frame with two or more blocks and >= 4096 compressed bytes in one submission and no dictionary: what makes a
    frame eligible for k_exec_cta (plan.h).  Eight Compressed blocks of about 3 KB each; at 65536 the lead frame and the first
    block fill one submission, and then every submission holds two blocks of the frame."""
    out = []
    for n in (8, 9):
        blocks, pos = [E.prefix(rng, 200)], 200
        for _ in range(n):
            s = _ordinary(rng, 120, pos, of_max=pos)
            b = E.Blk(bytes(rng.randrange(256) for _ in range(sum(q[0] for q in s) + 2600)), "raw", seqs=s, modes=[("pre",)] * 3)
            blocks.append(b)
            pos += _nominal([b])
        out.append(_ent("cta-shape", f"{n}-blocks-of-3KB", blocks, lead=64))
    return out


def append_block(frame, data):
    """`frame` with a Raw block of `data` after its last block (that block's Last_Block flag cleared; the checksum, if any, kept
    behind the new block)."""
    blocks = frame_blocks(frame)
    _, hl, _, checksum = frame_header(frame)
    start = blocks[-2][0] if len(blocks) > 1 else hl
    end = len(frame) - (4 if checksum else 0)
    h = int.from_bytes(frame[start:start + 3], "little") & ~1
    return (bytes(frame[:start]) + h.to_bytes(3, "little") + bytes(frame[start + 3:end]) + (1 | (len(data) << 3)).to_bytes(3, "little") +
            bytes(data) + bytes(frame[end:]))


def errors_after_cut(cs):
    """The crafted error cases of seqcraft and entcraft whose failing block is not the frame's first (each of them fails in its
    last block), with a Raw block appended after it: at 4096 the failing block is alone in its submission, right after a cut,
    and the frame goes on past it, so the next submission is already in flight and must start failed."""
    out = []
    tail = b"after the failing block " * 4
    for c in cs:
        if c.valid or len(c.blocks) < 2 or c.kind not in ("seq", "ent") or deviation(c):
            continue
        n = Case("errors-after-cut", c.id.split("-", 1)[1], "spliced", c, append_block(c.frame, tail), c.blocks + [("raw", tail)], ERROR,
                 dicts=c.dicts, dict_raw=c.dict_raw)
        n.fail_block, n.origin = len(c.blocks) - 1, c
        out.append(n)
    return out


FAMILIES = {"carry-tables": carry_tables, "carry-history": carry_history, "tail-reach": tail_reach, "alignment": alignment,
            "cta-shape": cta_shape}


def new_cases(crafted_cases=None):
    """The stream-edge families, built from fixed seeds; the error family from the crafted error cases."""
    out = []
    for i, (g, fn) in enumerate(FAMILIES.items()):
        out += fn(random.Random(0x57C0 + i))
    return out + errors_after_cut(crafted_cases if crafted_cases is not None else crafted())


# ---------------------------------------------------------------------------------------------------------------------------
# streams of cases, and what each cut carries
# ---------------------------------------------------------------------------------------------------------------------------
def separator(chunk):
    """A skippable frame that always ends the submission in front of it below the default chunk (it is longer than the chunk)."""
    return skippable(chunk if chunk < DEFAULT else 3)


PHASE_PLAIN = b"\x5a"
# at these chunks a case without a lead frame gets a one-byte one, so that its first block shares a submission with it: a
# Compressed block of a 128 KiB window (65536) or a small block (32768) in front of the next cut shifts every later cut by one
# block, and a frame of four or more blocks then has a submission that resumes and continues it with two of its blocks
PHASE_CHUNKS = (32768, 65536)


def stream(cases, chunk, head=b"", for_cut=False):
    """(bytes, the plaintext of the valid cases in order, [(case, offset of its frame, its lead frame, the lead's plaintext)]) of
    `cases` laid out for `chunk`.  for_cut: with every Dictionary_ID set to 0, so that the cut model, which has no dictionaries,
    cuts the stream as the decoder does."""
    parts, plain, at, pos = [head], bytearray(), [], len(head)
    for c in cases:
        lead, lead_plain = (c.lead, c.lead_plain) if c.lead or chunk not in PHASE_CHUNKS else (lead_frame(PHASE_PLAIN), PHASE_PLAIN)
        for p in (separator(chunk), lead):
            parts.append(p)
            pos += len(p)
        at.append((c, pos, lead, lead_plain))
        parts.append(c.cut_frame if for_cut else c.frame)
        pos += len(c.frame)
        if c.valid:
            plain += lead_plain + c.expected
    return b"".join(parts), bytes(plain), at


def section_modes(content):
    """(literals type, number of sequences, (LL, OF, ML) modes or None) of a Compressed block's content (RFC 8878 3.1.1.3)."""
    lt, sf = content[0] & 3, (content[0] >> 2) & 3
    if lt in (0, 1):
        need = 1 if sf in (0, 2) else (2 if sf == 1 else 3)
        regen = content[0] >> 3 if sf in (0, 2) else int.from_bytes(content[:need], "little") >> 4
        upper = 1 if lt == 1 else regen
    else:
        need = 3 if sf <= 1 else (4 if sf == 2 else 5)
        upper = (int.from_bytes(content[:need], "little") >> (4 + {0: 10, 1: 10, 2: 14, 3: 18}[sf])) & ((1 << {0: 10, 1: 10, 2: 14, 3: 18}[sf]) - 1)
    q = content[need + upper:]
    if not q or q[0] == 0:
        return lt, 0, None
    n, hl = (q[0], 1) if q[0] < 128 else ((((q[0] - 128) << 8) + q[1], 2) if q[0] < 255 else (q[1] + (q[2] << 8) + 0x7F00, 3))
    m = q[hl]
    return lt, n, ((m >> 6) & 3, (m >> 4) & 3, (m >> 2) & 3)


def frame_blocks(frame):
    """[(end offset in the frame, block type, compressed bytes, table actions)] of every block.  Table actions: per table of
    TABLES, "huf" / "fse" / "rle" / "pre" when the block defines it, "use" when it reads the current one (Treeless, Repeat),
    absent when it leaves it alone."""
    _, hl, _, checksum = frame_header(frame)
    pos, out = hl, []
    while True:
        h = int.from_bytes(frame[pos:pos + 3], "little")
        t, size = (h >> 1) & 3, h >> 3
        body = frame[pos + 3:pos + 3 + (1 if t == 1 else size)]
        pos += 3 + (1 if t == 1 else size)
        act = {}
        if t == 2:
            lt, n, modes = section_modes(body)
            if lt == 2:
                act["huf"] = "huf"
            elif lt == 3:
                act["huf"] = "use"
            for tab, m in zip(("ll", "of", "ml"), modes or ()):
                act[tab] = ("pre", "rle", "fse", "use")[m]
        if h & 1:
            pos += 4 if checksum else 0
        out.append((pos, t, len(body), act))
        if h & 1:
            return out


class Carry:
    """What one cut carries of a frame: P its plaintext before the cut, T the tail, residue the tail's source address mod 16
    (the output buffer is 16-byte aligned), unhashed P mod 32, resumed whether the frame was frame 0 of the submission before the
    cut, out_off where that submission placed it, tables {table: (kind, mode)} of the references its next block reads (kind:
    "slot" = built in the submission before the cut and copied, "carry" = already in the carry slot, "predefined",
    "dictionary", "none"), next_block its index."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def __repr__(self):
        return f"Carry({self.__dict__})"


def carries(cases, chunk, subs=None):
    """{case id: [Carry, ...]} over the stream of `cases` at `chunk` (subs: its cuts, streamcut.cut's by default); also returns
    {case id: [(submission index, its blocks of the case)]}."""
    data, _, at = stream(cases, chunk, for_cut=True)
    if subs is None:
        subs = streamcut.cut(data, chunk)[0]
    ends = [s[1] for s in subs]

    def sub_of(off):
        return next(i for i, e in enumerate(ends) if off <= e)
    # every frame in stream order: (case or None for a lead, start, [(end, type, csize, actions, size)])
    frames = []
    for c, pos, lead, lead_plain in at:
        if lead:
            lb = frame_blocks(lead)
            frames.append((None, pos - len(lead), [(pos - len(lead) + e, t, n, a, len(lead_plain)) for e, t, n, a in lb]))
        fb = frame_blocks(c.frame)
        frames.append((c, pos, [(pos + e, t, n, a, c.sizes[i]) for i, (e, t, n, a) in enumerate(fb)]))
    out, spans = {}, {}
    placed = {}      # submission -> bytes placed so far
    for c, start, blocks in frames:
        P, T, prev_sub = 0, 0, None
        # per table: its kind as the next submission would see it, and the mode that defined it
        dct = c is not None and c.tables0 == "dictionary"
        kinds = {t: "dictionary" for t in TABLES} if dct else {}
        modes = {t: "dict" for t in TABLES} if dct else {}
        seen = []
        for k, (end, t, csize, act, size) in enumerate(blocks):
            s = sub_of(end)
            if prev_sub is not None and s != prev_sub:
                # a cut in front of block k: the frame continued out of submission prev_sub
                W = c.window if c is not None else 1 << 20
                Tn = min(P, keep(W))
                off, produced = span
                used = {tab: (kinds.get(tab, "none"), modes.get(tab)) for tab, a in act.items() if a == "use"}
                if c is not None:
                    out.setdefault(c.id, []).append(Carry(P=P, T=Tn, keep=keep(W), residue=(off + produced - Tn) % 16, unhashed=P % 32,
                                                          resumed=off == 0 and resumed, out_off=off, tables=used, next_block=k,
                                                          next_size=size, sub=s))
                # the tables move into the carry: those built in the submission before the cut are copied (slot) and then
                # kept; predefined and dictionary tables are re-pointed
                kinds = {tab: ("carry" if kd == "slot" else kd) for tab, kd in kinds.items()}
                resumed, T = True, Tn
                span = (0, T)
            elif prev_sub is None:
                resumed = False
                span = (placed.get(s, 0), 0)
            if k == 0 or s != prev_sub:
                seen.append((s, []))
            seen[-1][1].append(k)
            for tab, a in act.items():
                if a != "use":
                    kinds[tab], modes[tab] = "predefined" if a == "pre" else "slot", a
            P += size
            off, produced = span
            span = (off, produced + size)
            placed[s] = off + produced + size
            prev_sub = s
        if c is not None:
            spans[c.id] = seen
    return out, spans
