"""Crafted invalid zstd frames, one fault each, and the census of the decoder's error leaves.

Every decoding leaf of b200z_error (include/b200zstd.h, codes 1-121, 200 and 210) is classified here, in plain Python with no
library call:
  - a crafted case below reaches it (`Case.leaf`, `dictionaries()`);
  - COVERED_ELSEWHERE: an existing test reaches it (API-level leaves, table errors of the entcraft / seqcraft / dictcraft sets);
  - UNREACHABLE: neither the reference nor the library can raise it, with the oracle line (oracle/ruzstd_oracle.c) and the ruzstd
    source line (ruzstd/src/..., crate ruzstd 0.9.1) that show why;
  - NOT_TESTED: reachable, but not by any test yet, and why.
The oracle's REFERENCE_WOULD_PANIC sites are classified the same way in PANIC_SITES, keyed by their line in ruzstd_oracle.c; the\ntwo that a decode_blocks call after an error reaches have a case in `reentries()`.

A case is a valid frame with one fault in it: the frame header cut short, a block body cut short, a literals section header,
a Huffman description, a literal stream or a sequence section's table modes broken.  Block faults come in two places: in the frame's
first block, and after a Raw block and a valid Compressed block (new Huffman table, FSE tables for LL / OF / ML, repeat offsets moved),
so the fault meets the tables and offsets an earlier block left behind.  Where the kernels have variants the cases cover each: direct
and FSE-compressed Huffman weights, 1 and 4 literal streams, a Treeless block, each of LL / OF / ML.  The list is fixed and seeded.

Stages are b200z_stage: 1 frame header, 3 block body (section headers, block reads), 4 literals, 5 sequences, 8 dictionary."""
import os
import random
import re
import struct

import entcraft as E
import seqcraft as S

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HEADER = os.path.join(ROOT, "include", "b200zstd.h")
ORACLE_C = os.path.join(ROOT, "oracle", "ruzstd_oracle.c")
FRAME_HEADER, BLOCK_BODY, LITERALS, SEQUENCES, DICTIONARY = 1, 3, 4, 5, 8


def decoding_leaves():
    """{name: code} of every decoding leaf of b200z_error: codes 1-121, 200 and 210 (the header is the source of truth)."""
    txt = open(HEADER).read()
    body = txt[txt.index("typedef enum b200z_error"):txt.index("} b200z_error;")]
    out = {}
    for name, v in re.findall(r"B200Z_ERR_([A-Z0-9_]+)\s*=\s*(\d+)", body):
        if 1 <= int(v) <= 121 or int(v) in (200, 210):
            out[name] = int(v)
    return out


def panic_lines():
    """Lines of oracle/ruzstd_oracle.c that return ZO_ERR_REFERENCE_WOULD_PANIC."""
    return [i + 1 for i, ln in enumerate(open(ORACLE_C)) if "return ZO_ERR_REFERENCE_WOULD_PANIC" in ln]


# ---------------------------------------------------------------------------------------------------------------------------
# frames
# ---------------------------------------------------------------------------------------------------------------------------
def block(kind, body, size=None, last=False):
    """One block: kind "raw" / "rle" / "cmp" with its body as given; `size` overrides the header's Block_Size (for a body cut short)."""
    t = {"raw": 0, "rle": 1, "cmp": 2}[kind]
    n = size if size is not None else (body[1] if kind == "rle" else len(body))
    head = struct.pack("<I", int(last) | (t << 1) | (n << 3))[:3]
    return head + (bytes([body[0]]) if kind == "rle" else bytes(body))


def frame_header(window_log=17):
    return struct.pack("<IBB", 0xFD2FB528, 0, (window_log - 10) << 3)


class Case:
    """One crafted invalid frame.  leaf / stage: what the reference raises; prefix_plain: the plaintext of the blocks before the
    faulty one; error_block / fault_at: the faulty block's index and its offset in the frame; at_end: the fault is the input ending (a frame cut short), so the frame can
    only be the last one of a buffer; libzstd: whether libzstd rejects it too (False marks a reference quirk); block_level: the fault
    lies past the section headers, where the block batch entry (b200z_decode_blocks_batch) can be handed it."""

    def __init__(self, name, data, leaf, stage, prefix_plain=b"", error_block=0, at_end=False, libzstd=True, block_level=False, fault_at=0):
        self.id, self.frame, self.leaf, self.stage, self.fault_at = name, bytes(data), leaf, stage, fault_at
        self.prefix_plain, self.error_block, self.at_end = bytes(prefix_plain), error_block, at_end
        self.libzstd, self.block_level = libzstd, block_level
        self.cap = len(self.prefix_plain) + S.BLOCK_MAX + 1024

    def __repr__(self):
        return self.id


class Earlier:
    """The valid blocks a "later" fault comes after: a Raw block, then a Compressed block with a new Huffman table (direct or
    FSE-compressed weights), FSE tables for LL / OF / ML and sequences that move the repeat offsets."""

    def __init__(self, rng, huf):
        self.huf = huf
        raw = E.prefix(rng, 64)
        modes = [("fse", 6, E.rand_norm(rng, 20, 6, neg=1, keep=(0, 1, 2, 3))), ("fse", 5, E.rand_norm(rng, 8, 5, neg=1, keep=(0, 1, 2, 3))),
                 ("fse", 6, E.rand_norm(rng, 24, 6, neg=1, keep=(0, 1, 2)))]
        cmp = E.seq_block(rng, modes, 40, pos=64, lit_mode="huf", huf=huf)
        self.state = {"huf": None, "ll": None, "of": None, "ml": None}
        content, _ = E.block_content(cmp, self.state)
        self.bytes = block("raw", raw[1]) + block("cmp", content)
        self.plain = S.execute(E.plain_blocks([raw, cmp]), ov=True)
        assert self.plain is not S.ERROR


def _frames(name, faulty, earlier, leaf, stage, **kw):
    """The first-block and the later-block frame of one faulty block (`faulty(state)` -> the block's bytes, header included)."""
    out = [Case(f"{name}-first", frame_header() + faulty(None), leaf, stage, fault_at=len(frame_header()), **kw)]
    if earlier is not None:
        st = dict(earlier.state)
        out.append(Case(f"{name}-later", frame_header() + earlier.bytes + faulty(st), leaf, stage, prefix_plain=earlier.plain,
                        error_block=2, fault_at=len(frame_header()) + len(earlier.bytes), **kw))
    return out


def huf_decode_stream(table, data):
    """(symbols, landed exactly) of one Huffman literal stream: the plain model of the reference's stream loop
    (literals_section_decoder.rs:94-146): after the padding, a state of max_bits bits, then per symbol its code length in bits,
    bits past the stream's start reading as zeros, until no more than -max_bits bits remain."""
    mb, entries = table
    assert data and data[-1]
    v, p = int.from_bytes(data, "little"), len(data) * 8 - (9 - data[-1].bit_length())

    def get(nb):
        nonlocal p
        p -= nb
        return ((v << max(0, -p)) >> max(0, p)) & ((1 << nb) - 1)
    state, out = get(mb), []
    while p > -mb:
        s, nb = entries[state]
        out.append(s)
        state = ((state << nb) & ((1 << mb) - 1)) | get(nb)
    return out, p == -mb


def overshooting_stream(table, lits):
    """A literal stream that decodes `lits` shifted by a few leading bits and overruns its start: the last code read takes more
    bits than the stream had left (LIT_BITSTREAM_READ_MISMATCH on a 4-stream section)."""
    mb, entries = table
    code = {}
    for i, (s, nb) in enumerate(entries):
        code.setdefault(s, (i >> (mb - nb), nb))
    for k in range(2 * len(lits) - 1):
        part = lits[k:] if k < len(lits) else lits[:2 * len(lits) - k - 1]
        for extra in range(1, mb):
            for val in range(1 << extra):
                w = E.BitW()
                for b in reversed(part):
                    w.add(*code[b])
                w.add(val, extra)
                s = w.backward()
                if not huf_decode_stream(table, s)[1]:
                    return s
    raise AssertionError("no overshooting stream for this table")


def _raw_lits(n=12):
    return E.lit_header(0, n) + bytes(range(0x41, 0x41 + n))


def cases():
    """The crafted invalid frames, from a fixed seed."""
    rng = random.Random(0xE4C0)
    out = []
    direct = E.Huf(E.lengths_for(rng, range(24), 6))
    fse = E.fse_weights(rng, E.lengths_for(rng, range(40), 7), 6, 1)
    assert direct.desc[0] == "direct" and fse.desc[0] == "fse"
    earlier = {"direct": Earlier(rng, direct), "fse": Earlier(rng, fse)}
    ed = earlier["direct"]

    # --- frame header cut short (stage 1): read_frame_header, frame.rs:6-85
    fh = struct.pack("<IBB", 0xFD2FB528, 3, 7 << 3) + struct.pack("<I", 0x1234)          # 4-byte dictionary id
    for cut in (0, 2):
        out.append(Case(f"dictionary-id-read-cut{cut}", fh[:6 + cut], "DICTIONARY_ID_READ", FRAME_HEADER, at_end=True))
    fh = struct.pack("<IBB", 0xFD2FB528, 2 << 6, 7 << 3) + struct.pack("<I", 5000)       # 4-byte content size
    for cut in (0, 3):
        out.append(Case(f"content-size-read-cut{cut}", fh[:6 + cut], "FRAME_CONTENT_SIZE_READ", FRAME_HEADER, at_end=True))
    out.append(Case("content-size-read-single-segment", struct.pack("<IB", 0xFD2FB528, 1 << 5), "FRAME_CONTENT_SIZE_READ",
                    FRAME_HEADER, at_end=True))
    fh = struct.pack("<IBB", 0xFD2FB528, 1 | (3 << 6), 7 << 3) + b"\x09" + struct.pack("<Q", 5000)  # 1-byte id, 8-byte size
    out.append(Case("content-size-read-8-bytes-after-dictionary-id", fh[:7 + 5], "FRAME_CONTENT_SIZE_READ", FRAME_HEADER, at_end=True))

    # --- a Raw or RLE block's body cut short (stage 3): decode_block_content, block_decoder.rs:55-72
    out += _frames("raw-body-cut", lambda st: block("raw", bytes(40), size=300, last=True), ed, "BLOCK_BODY_READ", BLOCK_BODY,
                   at_end=True)
    out += _frames("rle-body-missing", lambda st: struct.pack("<I", 1 | (1 << 1) | (50 << 3))[:3], ed, "BLOCK_BODY_READ", BLOCK_BODY,
                   at_end=True)

    # --- literals section header (stage 3): LiteralsSection::parse_from_header, literals_section.rs:117-223
    out += _frames("litsec-empty-block", lambda st: block("cmp", b"", last=True), ed, "LITSEC_GET_BITS", BLOCK_BODY)
    for name, content in (("raw-2-byte-size-in-1", b"\x04"), ("rle-3-byte-size-in-2", b"\x0d\x01"),
                          ("compressed-3-byte-header-in-1", b"\x02"), ("compressed-4-streams-3-byte-header-in-2", b"\x06\x10"),
                          ("compressed-4-byte-header-in-3", b"\x0a\x10\x00"), ("treeless-5-byte-header-in-4", b"\x0f\x10\x00\x00")):
        out += _frames(f"litsec-{name}", lambda st, c=content: block("cmp", c, last=True), ed, "LITSEC_NOT_ENOUGH_BYTES", BLOCK_BODY)

    # --- Huffman descriptions (stage 4): HuffmanTable::build_decoder / read_weights / build_table_from_weights, huff0_decoder.rs
    def huf_block(desc, regen=12, streams=1, payload=b"\x01"):
        """A Compressed block whose literals carry `desc` (bytes) and `payload`, then no sequences."""
        body = desc + payload
        return E.lit_header(2, regen, len(body), streams) + body + b"\x00"
    for streams in (1, 4):
        s = f"{streams}stream"
        out += _frames(f"huf-source-is-empty-{s}", lambda st, n=streams: block("cmp", E.lit_header(2, 12, 0, n) + b"\x00", last=True),
                       ed, "HUF_SOURCE_IS_EMPTY", LITERALS, block_level=True)
        out += _frames(f"huf-direct-40-weights-in-3-bytes-{s}", lambda st, n=streams: block("cmp", huf_block(bytes([127 + 40, 0x11, 0x22, 0x33]), streams=n, payload=b""), last=True),
                       ed, "HUF_NOT_ENOUGH_BYTES_IN_SOURCE", LITERALS, block_level=True)
        out += _frames(f"huf-direct-all-weights-zero-{s}", lambda st, n=streams: block("cmp", huf_block(bytes([127 + 3, 0, 0]), streams=n, payload=bytes(8)), last=True),
                       ed, "HUF_MISSING_WEIGHTS", LITERALS, block_level=True)
        zero = E.write_huf_desc([0] * 9, ("fse", 5, [31, 1]))
        out += _frames(f"huf-fse-all-weights-zero-{s}", lambda st, n=streams, d=zero: block("cmp", huf_block(d, streams=n, payload=bytes(8)), last=True),
                       ed, "HUF_MISSING_WEIGHTS", LITERALS, block_level=True)
        # one weight value at probability 32/32: every state reads 0 bits, so the weight stream never ends
        endless = E.write_ncount([0, 32], 5)
        w = E.BitW(); w.add(0, 5); w.add(0, 5)
        endless = bytes([len(endless) + 2]) + endless + w.backward()
        out += _frames(f"huf-fse-too-many-weights-{s}", lambda st, n=streams, d=endless: block("cmp", huf_block(d, streams=n, payload=bytes(8)), last=True),
                       ed, "HUF_TOO_MANY_WEIGHTS", LITERALS, block_level=True)
        good = fse.bytes()
        padded = bytes([good[0] + 1]) + good[1:] + b"\x00"                                      # weight stream ends in a zero byte
        out += _frames(f"huf-fse-weights-extra-padding-{s}", lambda st, n=streams, d=padded: block("cmp", huf_block(d, streams=n, payload=bytes(8)), last=True),
                       earlier["fse"], "HUF_EXTRA_PADDING", LITERALS, block_level=True)

    # --- literal streams (stage 4): a 4-stream section whose first or last stream overruns its start, literals_section_decoder.rs:128-146
    for wname, h in (("direct", direct), ("fse", fse)):
        lits = E.literals(rng, h.lengths, 64)
        for k in (0, 3):
            parts = [E.huf_stream(h.table, lits[16 * i:16 * (i + 1)]) for i in range(4)]
            parts[k] = overshooting_stream(h.table, lits[16 * k:16 * (k + 1)])
            pay = struct.pack("<3H", *(len(p) for p in parts[:3])) + b"".join(parts)

            def faulty(st, h=h, pay=pay, lits=lits):
                b = E.Blk(lits, "huf", huf=h, streams=4, raw={"lit_payload": pay})
                return block("cmp", E.block_content(b, dict(st or {"huf": None, "ll": None, "of": None, "ml": None}))[0], last=True)
            out += _frames(f"lit-stream{k}-overruns-{wname}-weights", faulty, earlier[wname], "LIT_BITSTREAM_READ_MISMATCH", LITERALS,
                           block_level=True)
        # Treeless: the stream is read with the table the earlier block left
        parts = [E.huf_stream(h.table, lits[16 * i:16 * (i + 1)]) for i in range(4)]
        parts[1] = overshooting_stream(h.table, lits[16:32])
        pay = struct.pack("<3H", *(len(p) for p in parts[:3])) + b"".join(parts)
        st = dict(earlier[wname].state)
        content = E.block_content(E.Blk(lits, "treeless", streams=4, raw={"lit_payload": pay}), st)[0]
        out.append(Case(f"lit-stream1-overruns-treeless-after-{wname}-weights-later", frame_header() + earlier[wname].bytes + block("cmp", content, last=True),
                        "LIT_BITSTREAM_READ_MISMATCH", LITERALS, prefix_plain=earlier[wname].plain, error_block=2, block_level=True,
                        fault_at=len(frame_header()) + len(earlier[wname].bytes)))

    # --- sequence section table modes (stage 5): an RLE mode whose byte is missing, sequence_section_decoder.rs:305-407
    # (tag, modes byte, the table bytes present): the missing byte alone, and after the earlier tables' RLE bytes
    for kind, leaf, modes in (("ll", "SEQ_MISSING_BYTE_FOR_RLE_LL_TABLE", [("", 1 << 6, b"")]),
                              ("of", "SEQ_MISSING_BYTE_FOR_RLE_OF_TABLE", [("", 1 << 4, b""), ("-after-rle-ll", (1 << 6) | (1 << 4), b"\x05")]),
                              ("ml", "SEQ_MISSING_BYTE_FOR_RLE_ML_TABLE", [("", 1 << 2, b""), ("-after-rle-ll-of", 0x54, b"\x05\x02")])):
        for tag, m, tables in modes:
            out += _frames(f"seq-rle-{kind}-byte-missing{tag}", lambda st, m=m, t=tables: block("cmp", _raw_lits() + b"\x03" + bytes([m]) + t, last=True),
                           ed, leaf, SEQUENCES, block_level=True)
    return out


def dictionaries():
    """((name, raw dictionary, leaf) of dictionaries Dictionary::decode_dict (dictionary.rs:45-126) rejects, the valid dictionary they
    come from): cut short in the magic number and ID, in the Huffman description, in each FSE description and in the repeat offsets,
    or with a bad magic number."""
    rng = random.Random(0xD1C7)
    h = E.Huf(E.lengths_for(rng, range(30), 7))
    of = (6, E.rand_norm(rng, 20, 6, neg=1, keep=(2, 3)))
    ml = (6, E.rand_norm(rng, 30, 6, neg=1, keep=(0, 1)))
    ll = (6, E.rand_norm(rng, 22, 6, neg=1, keep=(0, 1)))
    raw, _ = E.dictionary(0x4242, h, of, ml, ll, (1, 4, 8), bytes(rng.randrange(256) for _ in range(200)))
    hl = len(h.bytes())
    ends = [8 + hl]
    for log, norm in (of, ml, ll):
        ends.append(ends[-1] + len(E.write_ncount(norm, log)))
    out = [("empty", b"", "DICT_NOT_ENOUGH_BYTES"), ("7-bytes", raw[:7], "DICT_NOT_ENOUGH_BYTES"),
           ("bad-magic", bytes([raw[0] ^ 0xFF]) + raw[1:], "DICT_BAD_MAGIC_NUM"),
           ("bad-magic-8-bytes", raw[:3] + bytes([raw[3] ^ 1]) + raw[4:8], "DICT_BAD_MAGIC_NUM")]
    out.append(("no-huffman-table", raw[:8], "HUF_SOURCE_IS_EMPTY"))
    out.append(("cut-in-huffman-weights", raw[:8 + hl // 2], "HUF_NOT_ENOUGH_BYTES_IN_SOURCE"))
    for k, kind in enumerate(("of", "ml", "ll")):                # the FSE descriptions, in the order the dictionary holds them
        out.append((f"cut-in-{kind}-description", raw[:ends[k] + 1], "FSE_GET_BITS"))
    out.append(("cut-in-repeat-offsets", raw[:ends[3] + 7], "DICT_NOT_ENOUGH_BYTES"))
    out.append(("no-repeat-offsets", raw[:ends[3]], "DICT_NOT_ENOUGH_BYTES"))
    return out, raw


def good_frames():
    """Valid frames to put around the faulty ones: (frame, plaintext)."""
    rng = random.Random(0x600D)
    out = []
    for i in range(3):
        h = E.Huf(E.lengths_for(rng, range(16 + 8 * i), 5 + i))
        b0 = E.seq_block(rng, [("pre",)] * 3, 30, pos=64, lit_mode="huf", huf=h)
        blocks = [E.prefix(rng, 64), b0]
        data, _ = E.frame(blocks)
        out.append((data, S.execute(E.plain_blocks(blocks), ov=True)))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# the census
# ---------------------------------------------------------------------------------------------------------------------------
# leaf -> the test that reaches it (on the GPU and against the oracle)
COVERED_ELSEWHERE = {
    "MAGIC_NUMBER_READ": "tests/test_gpu_parity.py::test_truncation_sweep_matches_oracle",
    "BAD_MAGIC_NUMBER": "tests/test_gpu_parity.py::test_fuzz_artifacts_status_parity",
    "FRAME_DESCRIPTOR_READ": "tests/test_gpu_parity.py::test_truncation_sweep_matches_oracle",
    "WINDOW_DESCRIPTOR_READ": "tests/test_gpu_parity.py::test_truncation_sweep_matches_oracle",
    "SKIP_FRAME": "tests/test_host_units.py::test_frame_header_parse_matches_oracle_reset",
    "WINDOW_TOO_BIG": "tests/test_host_units.py::test_frame_header_parse_matches_oracle_reset",
    "WINDOW_SIZE_TOO_BIG": "tests/test_gpu_parity.py::test_fuzz_artifacts_status_parity",
    "DICT_NOT_PROVIDED": "tests/test_gpu_parity.py::test_fuzz_artifacts_status_parity",
    "NOT_YET_INITIALIZED": "tests/test_gpu_errcraft.py::test_frame_decoder_before_init",
    "FAILED_TO_READ_CHECKSUM": "tests/test_gpu_parity.py::test_fuzz_artifacts_status_parity",
    "FAILED_TO_DRAIN_DECODEBUFFER": "tests/test_gpu_decode_all_stream.py::test_failing_source_and_drain",
    "FAILED_TO_SKIP_FRAME": "tests/test_gpu_parity.py::test_api_decode_all",
    "TARGET_TOO_SMALL": "tests/test_gpu_parity.py::test_target_too_small_and_capacity_isolation",
    "BLOCK_HEADER_READ": "tests/test_gpu_parity.py::test_truncation_sweep_matches_oracle",
    "FOUND_RESERVED_BLOCK": "tests/test_gpu_parity.py::test_bitflip_sweep_matches_oracle",
    "BLOCK_SIZE_TOO_LARGE": "tests/test_gpu_parity.py::test_bitflip_sweep_matches_oracle",
    "BLOCK_CONTENT_READ": "tests/test_gpu_parity.py::test_truncation_sweep_matches_oracle",
    "MALFORMED_SECTION_HEADER": "tests/test_gpu_parity.py::test_bitflip_sweep_matches_oracle",
    "SEQHDR_NOT_ENOUGH_BYTES": "tests/test_gpu_parity.py::test_fuzz_artifacts_status_parity",
    "LIT_UNINITIALIZED_HUFFMAN_TABLE": "tests/test_gpu_entropy.py::test_entropy_one_batch",
    "LIT_MISSING_BYTES_FOR_JUMP_HEADER": "tests/test_gpu_entropy.py::test_entropy_one_batch",
    "LIT_MISSING_BYTES_FOR_LITERALS": "tests/test_gpu_entropy.py::test_entropy_one_batch",
    "LIT_EXTRA_PADDING": "tests/test_gpu_entropy.py::test_entropy_one_batch",
    "LIT_DECODED_LITERAL_COUNT_MISMATCH": "tests/test_gpu_parity.py::test_fuzz_artifacts_status_parity",
    "HUF_NOT_ENOUGH_BYTES_FOR_WEIGHTS": "tests/test_gpu_entropy.py::test_entropy_one_batch",
    "HUF_LEFTOVER_NOT_POWER_OF_2": "tests/test_gpu_entropy.py::test_entropy_one_batch",
    "HUF_FSE_TABLE_USED_TOO_MANY_BYTES": "tests/test_gpu_entropy.py::test_entropy_one_batch",
    "HUF_WEIGHT_BIGGER_THAN_MAX_NUM_BITS": "tests/test_gpu_entropy.py::test_entropy_one_batch",
    "HUF_MAX_BITS_TOO_HIGH": "tests/test_gpu_entropy.py::test_entropy_one_batch",
    "FSE_ACC_LOG_TOO_BIG": "tests/test_gpu_entropy.py::test_entropy_one_batch",
       "FSE_TOO_MANY_SYMBOLS": "tests/test_gpu_entropy.py::test_entropy_one_batch",
    "FSE_TABLE_IS_UNINITIALIZED": "tests/test_gpu_entropy.py::test_entropy_one_batch",
    "SEQ_EXTRA_PADDING": "tests/test_gpu_parity.py::test_bitflip_sweep_matches_oracle",
    "SEQ_NOT_ENOUGH_BYTES_FOR_NUM_SEQUENCES": "tests/test_gpu_parity.py::test_bitflip_sweep_matches_oracle",
    "SEQ_EXTRA_BITS": "tests/test_gpu_parity.py::test_bitflip_sweep_matches_oracle",
    "EXEC_NOT_ENOUGH_BYTES_FOR_SEQUENCE": "tests/test_gpu_crafted.py::test_crafted_one_batch",
    "EXEC_ZERO_OFFSET": "tests/test_gpu_crafted.py::test_crafted_one_batch",
    "EXEC_OFFSET_TOO_BIG": "tests/test_gpu_crafted.py::test_crafted_one_batch",
    "EXEC_NOT_ENOUGH_BYTES_IN_DICTIONARY": "tests/test_gpu_dictcraft.py::test_dictcraft_one_batch",
}

# leaf -> why no test reaches it yet
NOT_TESTED = {
    "BLOCK_OUTPUT_LIMIT": "the oracle raises it when one block's sequences add up past 2^31 bytes (ruzstd_oracle.c:891, where ruzstd's "
                          "u32 sum in sequence_execution.rs:44-52 would wrap and fail its assert): a 2 GiB block output.  The library's "
                          "other use, a Compressed block that decodes past its bound in decode_all_stream, is a documented deviation "
                          "(include/b200zstd.h, tier 1d) with no crafted case yet.",
}

# leaf -> why neither side can raise it: the oracle line and the ruzstd line that make it so
UNREACHABLE = {
    "INVALID_FRAME_DESCRIPTOR": "frame.rs:213-240 returns FrameDescriptorError only for a 2-bit flag outside 0..3 (the `other` arms), "
                                "and a 2-bit field has no such value; the oracle's table lookups (ruzstd_oracle.c:606-615) have no error.",
    "WINDOW_TOO_SMALL": "window_base is 1 << (10 + exponent) >= 1024 = MIN_WINDOW_SIZE (common/mod.rs:10, frame.rs:122-136; "
                        "ruzstd_oracle.c:629-633), and a single-segment frame takes its content size without the check (frame.rs:117-119, "
                        "ruzstd_oracle.c:628).",
    "DECODER_STATE_IS_FAILED": "raised by BlockDecoder when its state is Failed (block_decoder.rs:47), but FrameDecoder makes a new "
                               "BlockDecoder in every call (frame_decoder.rs:317, :463), so the state is never seen; the oracle keeps no "
                               "such state and decodes each block it reads (ruzstd_oracle.c:1141-1144, :1201).",
    "EXPECTED_HEADER_OF_PREVIOUS_BLOCK": "block_decoder.rs:49 fires only when decode_block_content is called twice for one header; "
                                         "frame_decoder.rs:317-377 and :463-529 read a header before every block, as the oracle "
                                         "does (ruzstd_oracle.c:1141-1144).",
    "LITSEC_ILLEGAL_TYPE": "literals_section.rs:233 is the `other` arm of a match on a 2-bit field (:119) that already lists 0..3; "
                           "ruzstd_oracle.c:640 takes the type from two bits.",
    "LIT_MISSING_COMPRESSED_SIZE": "decompress_literals (literals_section_decoder.rs:48) runs only for Compressed / Treeless "
                                   "literals, for which parse_from_header always sets compressed_size (literals_section.rs:180-221); "
                                   "ruzstd_oracle.c:688 vs :652.",
    "LIT_MISSING_NUM_STREAMS": "as LIT_MISSING_COMPRESSED_SIZE: num_streams is set with it (literals_section.rs:180-221; "
                               "literals_section_decoder.rs:49; ruzstd_oracle.c:689 vs :651).",
    "LIT_GET_BITS": "the literal streams' reader calls get_bits without `?` (literals_section_decoder.rs:100, :132; huff0_decoder.rs:34, "
                    ":46): a read past the start gives zeros, never an error (ruzstd_oracle.c:669-686).",
    "HUF_GET_BITS": "read_weights reads its bits with BitReaderReversed::get_bits, which does not fail (huff0_decoder.rs:191, "
                    "fse_decoder.rs:43-51); the FSE description's own read errors surface as FSE_GET_BITS (ruzstd_oracle.c:244-268).",
    "HUF_FSE_DECODER": "init_state fails only on a table of accuracy log 0 (fse_decoder.rs:32-34), and the weights table was just "
                       "built with accuracy log 5 + a 4-bit field >= 5 (fse_decoder.rs:235-237; ruzstd_oracle.c:245, :347-348).",
    "HUF_NOT_ENOUGH_BYTES_TO_DECOMPRESS_WEIGHTS": "compressed_weights.len() = fse_stream.len() - used and compressed_length = header - "
                                                  "used, so the check (huff0_decoder.rs:177) is fse_stream.len() < header, which "
                                                  "NotEnoughBytesForWeights (:146) already rejected (ruzstd_oracle.c:335, :342).",
    "FSE_ACC_LOG_IS_ZERO": "the accuracy log read from a description is 5 + a 4-bit field (fse_decoder.rs:233-237, ruzstd_oracle.c:245-247) "
                           "and build_from_probabilities is called with the predefined logs 6, 5, 6 (sequence_section_decoder.rs:418-442, "
                           "ruzstd_oracle.c:288, :784-788).",
    "FSE_PROBABILITY_COUNTER_MISMATCH": "each count read is value - 1 with value <= max_remaining = remaining + 1 (bits_to_read = "
                                        "highest_bit_set(max_remaining), value = unchecked - low_threshold <= (2^bits - 1) - "
                                        "low_threshold = max_remaining; fse_decoder.rs:243-262), so the counter never passes the sum and "
                                        "the loop (:241) ends on equality; ruzstd_oracle.c:249-274.",
    "SEQ_UNSUPPORTED_OFFSET": "an offset code is a symbol of the OF table, whose symbols stop at MAX_OFFSET_CODE = 31 (FSETable::new("
                              "MAX_OFFSET_CODE), fse_decoder.rs:142 -> FSE_TOO_MANY_SYMBOLS), or an RLE byte, rejected above 31 "
                              "(sequence_section_decoder.rs:355); so of_code > 31 (:104, :179) never holds; ruzstd_oracle.c:775, :820.",
    "SEQ_ZERO_OFFSET": "offset = bits + (1 << of_code) with of_code <= 31 (see SEQ_UNSUPPORTED_OFFSET) is >= 1 and, with at most 31 "
                       "bits < 2^31, cannot wrap a u32 (sequence_section_decoder.rs:110-114, :185-189; ruzstd_oracle.c:823-824).",
    "SEQ_MISSING_COMPRESSION_MODE": "parse_from_header sets the modes byte whenever num_sequences != 0 (sequence_section.rs:108-167), and "
                                    "decode_sequences runs only then (block_decoder.rs:160-170, sequence_section_decoder.rs:301); "
                                    "ruzstd_oracle.c:730-747, :782, :968.",
}

# oracle line -> why the assert / unreachable!() / index it restates cannot fire, or how it is reached
PANIC_SITES = {
    202: "table size > FSE_MAX_TABLE: every accuracy log is capped at 9 before the build (ruzstd_oracle.c:246, fse_decoder.rs:238-240).",
    208: "more -1 counts than table cells: each -1 adds one to a counter that stops at the table size (fse_decoder.rs:264-266), "
         "so negative_idx reaches 0 only after the last one (fse_decoder.rs:156-163).",
    223: "the spread never lands below negative_idx: the step (size/2 + size/8 + 3) is odd, so it visits every cell "
         "(fse_decoder.rs:170-184), and some cell is below negative_idx whenever a count is positive.",
    233: "nb > accuracy log: nb = acc_log - floor(log2(count + k)) <= acc_log for count >= 1 (fse_decoder.rs:190-215).",
    305: "REACHED on re-entry: a description that fails with AccLogTooBig has already set accuracy_log (fse_decoder.rs:230-237, "
         "ruzstd_oracle.c:245-246) and left the cells as they were (none at a frame's start).  decode_blocks keeps no failed state "
         "(frame_decoder.rs:309-377, ruzstd_oracle.c:1135-1162), so a caller that calls it again after the error reads the next "
         "block; a Repeat mode there passes init_state's check (fse_decoder.rs:33) and indexes decode[] with accuracy_log bits "
         "(:37), past its cells.",
    312: "a state update past the table: baseline + 2^nb <= table size for every cell (fse_decoder.rs:190-215, :43-51).  A failed "
         "description changes accuracy_log but neither the cells nor decode_len (ruzstd_oracle.c:240-285), and a state reached from "
         "a cell stays inside that cell's table, so re-entry does not reach it either: a state outside the cells is caught at :305.",
    352: "the weights' state update is fsed_update_state, which can only fail at :312; its table was built in the same call, "
         "and bits past the stream's start read as zeros (bit_reader_reverse.rs get_bits_cold), never a panic (huff0_decoder.rs:212-226).",
    355: "as :352, for the second weights state (huff0_decoder.rs:219-226).",
    399: "rank_indexes[0] != table size (assert, huff0_decoder.rs:353): the weights' 2^(w-1) plus the implicit last weight's "
         "leftover sum to exactly 2^max_bits once the leftover is a power of two (:317-330).",
    677: "REACHED on re-entry: HuffmanTable::build_decoder clears the table (huff0_decoder.rs:118, ruzstd_oracle.c:412), then "
         "build_table_from_weights sets max_num_bits before it returns MaxBitsTooHigh (:322-325, ruzstd_oracle.c:390-391).  "
         "Called again after that error, decode_blocks reads the next block; a Treeless block passes the uninitialized check "
         "(literals_section_decoder.rs:61, ruzstd_oracle.c:697) and indexes the empty table.",
    756: "an LL code > 35: RLE codes above 35 are rejected (sequence_section_decoder.rs:319-321) and FSE tables hold symbols <= 35 "
         "(fse_decoder.rs:142).",
    763: "an ML code > 52: as :756 (sequence_section_decoder.rs:389-391, fse_decoder.rs:142).",
    830: "the LL state update can only fail at :312 (sequence_section_decoder.rs:198-200).",
    831: "the ML state update, as :830 (sequence_section_decoder.rs:198-200).",
    832: "the OF state update, as :830 (sequence_section_decoder.rs:198-200).",
    898: "seq_sum != bytes added (assert, sequence_execution.rs:47-52): every sequence adds exactly ll + ml bytes and the rest of the "
         "literals are added and counted (ruzstd_oracle.c:880-897); only a u32 wrap could break it, which :891 reports first.",
    955: "regenerated size != literals decoded (assert, block_decoder.rs:146): Raw and RLE push exactly that many, Compressed checks the "
         "count itself (LIT_DECODED_LITERAL_COUNT_MISMATCH, literals_section_decoder.rs:150-156).",
    956: "bytes used != the section's size (assert, block_decoder.rs:152): decompress_literals consumes compressed_size exactly, Raw "
         "regenerated_size and RLE one byte (literals_section_decoder.rs:58-158).",
}


class Reentry:
    """A frame whose first failing block leaves a half-built table behind, followed by a block that reads it.  FrameDecoder::
    decode_blocks keeps no failed state, so a second call after the first error decodes the next block and panics in the reference
    (REFERENCE_WOULD_PANIC at oracle line `site`).  The library does not go on: its decode_blocks returns the first error again until
    the decoder is reset (include/b200zstd.h, tier 2)."""

    def __init__(self, name, data, first, site):
        self.id, self.frame, self.first, self.site = name, bytes(data), first, site
        self.second = ("REFERENCE_WOULD_PANIC", first[1])

    def __repr__(self):
        return self.id


def reentries():
    desc, pay = bytes([127 + 2, 0xBB]), b"\x01\x02\x03\x80"                      # weights 11, 11: max_bits 12
    b0 = E.lit_header(2, 12, len(desc) + len(pay), 1) + desc + pay + b"\x00"
    b1 = E.lit_header(3, 12, 2, 1) + b"\x55\x80" + b"\x00"
    huf = Reentry("huf-max-bits-too-high-then-treeless", frame_header() + block("cmp", b0) + block("cmp", b1, last=True),
                  ("HUF_MAX_BITS_TOO_HIGH", LITERALS), 677)
    b0 = _raw_lits() + b"\x01" + bytes([2 << 6]) + bytes([10 - 5])                     # LL description at accuracy log 10 > 9
    b1 = _raw_lits() + b"\x01" + bytes([3 << 6]) + b"\x5a\x3c\x99\x01"             # LL Repeat
    fse = Reentry("ll-acc-log-too-big-then-repeat", frame_header() + block("cmp", b0) + block("cmp", b1, last=True),
                  ("FSE_ACC_LOG_TOO_BIG", SEQUENCES), 305)
    return [huf, fse]


def census():
    """{leaf: ("case", [case ids]) | ("test", test id) | ("unreachable", reason)} over every decoding leaf of the header."""
    reached = {}
    for c in cases():
        reached.setdefault(c.leaf, []).append(c.id)
    for name, _, leaf in dictionaries()[0]:
        reached.setdefault(leaf, []).append(f"dict-{name}")
    out = {}
    for leaf in decoding_leaves():
        if leaf in reached:
            out[leaf] = ("case", reached[leaf])
        elif leaf in COVERED_ELSEWHERE:
            out[leaf] = ("test", COVERED_ELSEWHERE[leaf])
        elif leaf in UNREACHABLE:
            out[leaf] = ("unreachable", UNREACHABLE[leaf])
        elif leaf in NOT_TESTED:
            out[leaf] = ("not tested", NOT_TESTED[leaf])
    out["REFERENCE_WOULD_PANIC"] = ("case", [r.id for r in reentries()])         # every other site is classified in PANIC_SITES
    return out
