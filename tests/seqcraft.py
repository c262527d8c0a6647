"""Crafted zstd frames with chosen sequences, shared by the CPU and GPU tests of the sequence and execution stages.

A frame is a list of blocks: ("raw", bytes), ("rle", byte, count) or ("cmp", literals, [(ll, ml, of), ...]).  The Compressed
blocks are written by zstd-rs_b200/csrc/encode.cuh compiled for the host (tests/host/encode_test.cpp), so a sequence can be
placed at any batch, row or word boundary of the execution kernels.  `of` is the actual offset, or -- in Offset_Value mode
(`ov=True`) -- the zstd Offset_Value itself, where 1-3 are repeat codes.

`execute` is the reference: plain LZ77 written from the format (RFC 8878 3.1.1.4-3.1.1.5), independent of the oracle and of
the kernels' models.  `cases()` builds the crafted set the tests run; each case's id names the kernel constant it sits on."""
import atexit
import os
import random
import shutil
import struct
import subprocess
import tempfile

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
HERE = os.path.dirname(os.path.abspath(__file__))
ERROR = "error"
BLOCK_MAX = 131072

# kernel constants the cases are placed around (zstd-rs_b200/csrc/kernels.cu, exec_cta.cuh)
EXEC_BATCH = 64          # k_exec: sequences per batch
EXEC_TMAX = 8128         # k_exec: most bytes one batch produces on its fast path
FSE_PUBLISH = 128        # k_fse: sequences between two progress publications
XC_BATCH = 1024          # k_exec_cta: sequences per batch
FSE_FAST_XBITS = 38      # k_fse: most extra bits (LL + ML + OF) one sequence may carry on the fast path
OVERLAP_LENGTHS = [3, 4, 31, 32, 33, 127, 128, 129, 300]

# k_exec_cta's reasons for handing a frame back to k_exec, as b200z_batch_debug_sched reports them (XC_WHY_* in exec_cta.cuh)
WHY_SEQ_RECORDS = 4      # raw offsets that cannot be resolved in place (values >= 2^30)
WHY_BLOCK_SIZE = 8       # block sizes / literal counts it does not take
WHY_SEQ_CHECK = 32       # sequence validation failed (offset 0, offset beyond the output)


_exe = None


def encoder():
    """Path of the host encoder, compiled once per process into a temporary directory."""
    global _exe
    if _exe is None:
        d = tempfile.mkdtemp(prefix="seqcraft")
        atexit.register(shutil.rmtree, d, True)
        exe = os.path.join(d, "encode_test")
        subprocess.check_call([NVCC, "-x", "cu", "-std=c++17", "-O2", "-w", "-o", exe, os.path.join(HERE, "host", "encode_test.cpp")])
        _exe = exe
    return _exe


def encode(lits, seqs, ov=False):
    """Content of a Compressed block for `lits` and `seqs`; returns (content, huffman literals 0/1, [LL, OF, ML] modes)."""
    exe = encoder()
    d = os.path.dirname(exe)
    src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    with open(src, "wb") as f:
        f.write(struct.pack("<I", len(lits)) + bytes(lits) + struct.pack("<I", len(seqs)) +
                b"".join(struct.pack("<3I", ll, ml, of & 0xFFFFFFFF) for ll, ml, of in seqs))
    out = subprocess.run([exe] + (["--ov"] if ov else []) + [src, dst], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.startswith("ok"), out.stdout + out.stderr
    f = out.stdout.split()
    with open(dst, "rb") as fh:
        return fh.read(), int(f[2]), [int(x) for x in f[3:6]]


def offset_history(ov, ll, h):
    """Offset_Value + literal length -> actual offset, updating the repeat-offset history h (RFC 8878 3.1.2.5)."""
    if ov > 3:
        actual = ov - 3
        h[:] = [actual, h[0], h[1]]
        return actual
    r = ov - 1 + (1 if ll == 0 else 0)     # with ll == 0 the repeat codes shift by one
    if r == 0:
        return h[0]
    actual = max(h[0] - 1, 0) if r == 3 else h[r]
    h[:] = [actual, h[0], h[2]] if r == 1 else [actual, h[0], h[1]]
    return actual


def execute(blocks, ov=False):
    """The frame's content, or ERROR.  History starts as [1, 4, 8] and carries across blocks; Raw and RLE blocks leave it
    alone.  Matches copy byte by byte, so an overlapping match repeats its last `offset` bytes."""
    out = bytearray()
    h = [1, 4, 8]
    for b in blocks:
        if b[0] == "raw":
            out += b[1]
        elif b[0] == "rle":
            out += bytes([b[1]]) * b[2]
        else:
            lits, seqs = b[1], b[2]
            li = 0
            for ll, ml, of in seqs:
                if li + ll > len(lits):
                    return ERROR
                out += lits[li:li + ll]
                li += ll
                off = offset_history(of if ov else of + 3, ll, h)
                if off == 0 or off > len(out):
                    return ERROR
                for _ in range(ml):
                    out.append(out[-off])
            out += lits[li:]
    return bytes(out)


def nominal_size(blocks):
    """Bytes the blocks would produce if every sequence executed (the output capacity given to error cases)."""
    n = 0
    for b in blocks:
        if b[0] == "raw":
            n += len(b[1])
        elif b[0] == "rle":
            n += b[2]
        else:
            n += len(b[1]) + sum(ml for _, ml, _ in b[2])
    return n


def frame(blocks, window_log=17, content_size=True, checksum=False, ov=False, plain=None, dict_id=None, dict_id_bytes=4,
          single_segment=False, window_desc=None):
    """The frame's bytes, and (huffman literals 0/1, [LL, OF, ML] modes) of each Compressed block.  content_size: True = the
    reference's content size (omitted for an error case), None = no Frame_Content_Size field, or a number.  checksum: append
    the content checksum (XXH64 of the reference's content).  plain: the content, when `execute` cannot tell it (a frame that
    reaches into a dictionary).  dict_id: a Dictionary_ID field of dict_id_bytes (1, 2 or 4) bytes.  single_segment: no
    Window_Descriptor, the window is the content size.  window_desc: the Window_Descriptor byte (exponent and mantissa)."""
    if plain is None:
        plain = execute(blocks, ov)
    if content_size is True:
        content_size = None if plain is ERROR else len(plain)
    fhd = (4 if checksum else 0)
    fcs = b""
    if content_size is not None:
        if single_segment and content_size < 256:
            fcs = struct.pack("<B", content_size)
        else:
            fcs = struct.pack("<I", content_size) if content_size < 1 << 32 else struct.pack("<Q", content_size)
            fhd |= (2 if len(fcs) == 4 else 3) << 6
    did = b""
    if dict_id is not None:
        did = struct.pack("<Q", dict_id)[:dict_id_bytes]
        assert int.from_bytes(did, "little") == dict_id
        fhd |= {1: 1, 2: 2, 4: 3}[dict_id_bytes]
    if single_segment:
        assert content_size is not None
        out = struct.pack("<IB", 0xFD2FB528, fhd | 0x20) + did + fcs
    else:
        wd = (window_log - 10) << 3 if window_desc is None else window_desc
        out = struct.pack("<IBB", 0xFD2FB528, fhd, wd) + did + fcs
    encs = []
    for i, b in enumerate(blocks):
        last = 1 if i + 1 == len(blocks) else 0
        if b[0] == "raw":
            assert len(b[1]) <= BLOCK_MAX
            out += struct.pack("<I", last | (len(b[1]) << 3))[:3] + bytes(b[1])
        elif b[0] == "rle":
            assert b[2] <= BLOCK_MAX
            out += struct.pack("<I", last | (1 << 1) | (b[2] << 3))[:3] + bytes([b[1]])
        else:
            assert len(b[1]) + sum(ml for _, ml, _ in b[2]) <= BLOCK_MAX
            content, huf, modes = encode(b[1], b[2], ov)
            encs.append((huf, modes))
            assert len(content) <= BLOCK_MAX
            out += struct.pack("<I", last | (2 << 1) | (len(content) << 3))[:3] + content
    if checksum:
        from oracle import oracle as O
        out += struct.pack("<I", O.xxh64(plain if plain is not ERROR else b"") & 0xFFFFFFFF)
    return out, encs


def oracle_decode(oracle, data, blocks, ov=False):
    """Decodes `data` with the oracle and checks that its trace holds exactly the requested sequences -- {ll, ml, Offset_Value}
    (trace columns 0-2) -- up to where it stopped.  Returns (content, None) or (None, (error leaf, stage))."""
    d = oracle.FrameDecoder()
    d.trace_enable()
    try:
        r = d.reset(data)
        d.decode_blocks(r, oracle.ALL)
        res = (d.collect(), None)
    except oracle.OracleError as e:
        res = (None, (oracle.error_names()[e.code].replace("ZO_", ""), e.stage))
    _, _, seqs = d.trace()
    want = [(ll, ml, of if ov else of + 3) for b in blocks if b[0] == "cmp" for ll, ml, of in b[2]]
    got = [tuple(int(x) for x in s[:3]) for s in seqs]
    assert got == want[:len(got)], "the oracle decoded other sequences than the ones requested"
    if res[1] is None:
        assert len(got) == len(want)
    return res


# ---------------------------------------------------------------------------------------------------------------------------
# the crafted cases
# ---------------------------------------------------------------------------------------------------------------------------
class Case:
    """One crafted frame.  handback: None = k_exec_cta must execute the whole frame itself; otherwise the reason bit it must
    report when it hands the frame to k_exec (only error cases do).  xbits: extra bits of the one wide sequence (k_fse group)."""

    def __init__(self, group, name, blocks, window_log=17, ov=False, handback=None, xbits=None):
        self.group, self.id = group, f"{group}-{name}"
        self.blocks, self.window_log, self.ov = blocks, window_log, ov
        self.handback, self.xbits = handback, xbits
        self.expected = execute(blocks, ov)
        self.valid = self.expected is not ERROR
        self.cap = len(self.expected) if self.valid else nominal_size(blocks)
        self._frame = None

    @property
    def frame(self):
        if self._frame is None:
            self._frame = frame(self.blocks, self.window_log, checksum=self.valid, ov=self.ov)[0]
        return self._frame

    def __repr__(self):
        return self.id


def skewed(rng, n, alphabet=b"abcdefghijklmnop"):
    return bytes(rng.choice(alphabet) for _ in range(n))


def _ordinary(rng, n, pos, ll_max=3, ml_lo=3, ml_hi=20, of_max=BLOCK_MAX):
    """n short sequences starting at output position pos (> 0): small literal runs and matches, offsets anywhere behind."""
    seqs = []
    for _ in range(n):
        ll, ml = rng.randint(0, ll_max), rng.randint(ml_lo, ml_hi)
        seqs.append((ll, ml, rng.randint(1, min(pos + ll, of_max))))
        pos += ll + ml
    return seqs


def _end(seqs):
    return sum(q[0] + q[1] for q in seqs)


def _cmp(rng, seqs, tail=0):
    return ("cmp", skewed(rng, sum(q[0] for q in seqs) + tail), seqs)


def geometry(rng):
    out = []
    names = {1: "one", 31: "EXEC_BATCH/2-1", 32: "EXEC_BATCH/2", 33: "EXEC_BATCH/2+1", 63: "EXEC_BATCH-1", 64: "EXEC_BATCH",
             65: "EXEC_BATCH+1", 127: "FSE_PUBLISH-1", 128: "FSE_PUBLISH", 129: "FSE_PUBLISH+1", 1023: "XC_BATCH-1",
             1024: "XC_BATCH", 1025: "XC_BATCH+1", 2049: "2*XC_BATCH+1"}
    for n, name in names.items():
        seqs = [(16, 5, 7)] + _ordinary(rng, n - 1, 21)
        out.append(Case("geometry", f"nseq{n}={name}", [_cmp(rng, seqs, tail=rng.randint(0, 9))]))
    # three batches of EXEC_BATCH sequences; the middle one produces EXEC_TMAX - 1, EXEC_TMAX or EXEC_TMAX + 1 bytes
    for d in (-1, 0, 1):
        first = [(100, 10, 50)] + _ordinary(rng, EXEC_BATCH - 1, 110)
        mid = [(27, 100, rng.randint(1, _end(first))) for _ in range(EXEC_BATCH)]
        mid[-1] = (27, 100 + d, 33)
        seqs = first + mid + _ordinary(rng, EXEC_BATCH, _end(first + mid))
        assert sum(q[0] + q[1] for q in mid) == EXEC_TMAX + d
        out.append(Case("geometry", f"batch-bytes{EXEC_TMAX + d}=EXEC_TMAX{d:+d}", [_cmp(rng, seqs, tail=5)]))
    seqs = [(40, 9, 30)] + _ordinary(rng, 20, 49) + [(3, EXEC_TMAX + 900, 17)]
    seqs += _ordinary(rng, 20, _end(seqs))
    out.append(Case("geometry", "one-seq-longer-than-EXEC_TMAX", [_cmp(rng, seqs, tail=3)]))
    return out


def overlap(rng):
    """Overlapping matches (offset < length) for every offset: each length starts at every residue mod 32 (so at every byte of
    k_exec's 32-byte rows and of a 4-byte word) and at each of the four 32-byte quarters of k_exec_cta's 128-byte rows.  Frames
    are laid out 128-byte aligned by the tests."""
    out = []
    for of in list(range(1, 41)) + [63, 64, 65, 127, 128, 129]:
        seqs, pos = [], 0
        for j, ml in enumerate(OVERLAP_LENGTHS):
            for r32 in range(32):
                res = r32 + 32 * ((j + r32 + of) % 4)
                ll = (res - pos) % 128
                while pos + ll < of:
                    ll += 128
                seqs.append((ll, ml, of))
                pos += ll + ml
        out.append(Case("overlap", f"of{of}-rows32-rows128", [_cmp(rng, seqs, tail=1)]))
    return out


def dense(rng):
    """ll = 0, ml = 3: the owner changes every 3 bytes, so 4-byte words span two sequences; sources in the same row / batch."""
    out = []
    for of in [3, 4, 6] + list(range(30, 41)) + list(range(60, 71)):
        seqs = [(128, 3, of)] + [(0, 3, of)] * 3000 + [(1, 3, of)] + [(0, 3, of)] * 100
        out.append(Case("dense", f"ll0-ml3-of{of}-words", [_cmp(rng, seqs, tail=2)]))
    return out


def earlier_blocks(rng):
    """Frames of 3-6 Compressed blocks with Raw / RLE blocks between them; matches reaching the frame start, the previous
    Compressed block and exactly the window."""
    out = []
    for ncmp, wlog, sep in ((3, 17, "raw"), (4, 17, "rle"), (5, 17, "both"), (6, 17, "raw"), (4, 16, "rle")):
        window = 1 << wlog
        blocks, pos, prev_cmp = [], 0, None
        for k in range(ncmp):
            if k and sep in ("raw", "both"):
                raw = bytes(rng.randrange(256) for _ in range(rng.randint(1, 3000)))
                blocks.append(("raw", raw)); pos += len(raw)
            if k and sep in ("rle", "both"):
                n = rng.randint(1, 5000)
                blocks.append(("rle", rng.randrange(256), n)); pos += n
            start = pos
            seqs = [(20, 4, min(pos + 20, 9))] if k == 0 else []
            p = pos + sum(q[0] + q[1] for q in seqs)
            budget = min(window, BLOCK_MAX) - 4000
            while p - start < budget - 400:
                r = rng.random()
                ll = rng.randint(0, 5)
                ml = rng.randint(3, 60)
                of = rng.randint(1, min(p + ll, window))
                if r < 0.05 and p + ll <= window:
                    of = p + ll                                   # the frame's first byte
                elif r < 0.10 and prev_cmp is not None and p + ll - prev_cmp[0] <= window:
                    of = p + ll - rng.randint(*prev_cmp)          # into the previous Compressed block
                elif r < 0.15 and p + ll >= window:
                    of = window                                   # exactly the window
                seqs.append((ll, ml, of))
                p += ll + ml
            blk = _cmp(rng, seqs, tail=rng.randint(0, 50))
            blocks.append(blk)
            pos = start + len(blk[1]) + sum(q[1] for q in seqs)
            prev_cmp = (start, pos - 1)
        uses_window = any(q[2] == window for b in blocks if b[0] == "cmp" for q in b[2])
        out.append(Case("earlier", f"cmp{ncmp}-{sep}-wlog{wlog}" + ("-of=window" if uses_window else ""), blocks, window_log=wlog))
    # an offset reaching exactly the frame's first byte, and one beyond it: in a frame shorter than its window (so only the
    # produced-bytes check can reject it) and in one that has produced more than its window
    lits = skewed(rng, 10)
    short = [_cmp(rng, [(30, 6, 4)] + _ordinary(rng, 200, 36)), ("rle", 0x5A, 700)]
    n = nominal_size(short)
    out.append(Case("earlier", "of=produced-inside-window", short + [("cmp", lits, [(10, 5, n + 10)])]))
    out.append(Case("earlier", "of=produced+1-inside-window", short + [("cmp", lits, [(10, 5, n + 11)])], handback=WHY_SEQ_CHECK))
    base = out[0].blocks
    produced = len(out[0].expected)
    out.append(Case("earlier", "of=produced+1", base + [("cmp", lits, [(10, 5, produced + 11)])], handback=WHY_SEQ_CHECK))
    out.append(Case("earlier", "sum-ll>literals", base + [("cmp", lits[:7], [(3, 5, 100), (5, 4, 9)])], handback=WHY_BLOCK_SIZE))
    return out


def cta_edges(rng):
    """Blocks of exactly 131072 bytes: the extremes of k_exec_cta's 18-bit record fields, and its global-literal mode."""
    out = []
    out.append(Case("cta-block", "litrun131069-ml3-XC_LITG_BIAS",
                    [("cmp", skewed(rng, BLOCK_MAX - 3), [(BLOCK_MAX - 3, 3, 7)])]))
    prev = ("raw", bytes(rng.randrange(256) for _ in range(BLOCK_MAX)))
    out.append(Case("cta-block", "ll0-match131072-of=window", [prev, ("cmp", b"", [(0, BLOCK_MAX, BLOCK_MAX)])]))
    out.append(Case("cta-block", "ll0-match131072-of65536", [prev, ("cmp", b"", [(0, BLOCK_MAX, 65536)])]))
    seqs = [(rng.randint(1, 9), 20000, rng.randint(1, 5000)) for _ in range(5)]
    tail = BLOCK_MAX - sum(q[0] + q[1] for q in seqs)
    out.append(Case("cta-block", f"5seqs-then-tail{tail}", [prev, _cmp(rng, seqs, tail=tail)]))
    seqs = [(40000, 3, 11), (40000, 5, 39999), (40000, 4, 2)]
    tail = BLOCK_MAX - sum(q[0] + q[1] for q in seqs)
    out.append(Case("cta-block", "nearly-all-literals-XC_LITG_BIAS", [_cmp(rng, seqs, tail=tail)]))
    for c in out:
        assert all(nominal_size([b]) == BLOCK_MAX for b in c.blocks)
    return out


def repeats(rng):
    """Offset_Value 1-3 (repeat codes) with ll = 0 and ll > 0: as the first sequence of a block (resolved against the history
    at the block's start), across Raw / RLE blocks and Compressed blocks without sequences; rep0 - 1 saturating to 0."""
    out = []
    head = ("cmp", skewed(rng, 40), [(20, 4, 13 + 3), (5, 4, 9 + 3), (5, 4, 17 + 3)])    # history [17, 9, 13]
    seps = {"none": [], "raw": [("raw", b"xyz" * 7)], "rle": [("rle", 0x41, 300)], "cmp0seq": [("cmp", skewed(rng, 30), [])]}
    for sep, mid in seps.items():
        for ov in (1, 2, 3):
            for ll in (0, 6):
                tail = [(ll, 5, ov), (0, 4, 1), (2, 6, 3), (0, 3, 2), (1, 7, 50 + 3), (0, 4, 3)]
                blocks = [head] + mid + [("cmp", skewed(rng, ll + 3), tail)]
                out.append(Case("repeat", f"ov{ov}-ll{ll}-first-after-{sep}", blocks, ov=True))
    # the history every frame starts with, [1, 4, 8]
    for ov, ll in ((1, 5), (2, 5), (3, 9), (1, 0)):
        blocks = [("cmp", skewed(rng, ll + 2), [(ll, 6, ov), (0, 3, 1)])]
        out.append(Case("repeat", f"ov{ov}-ll{ll}-initial-history", blocks, ov=True,
                        handback=None if execute(blocks, True) is not ERROR else WHY_SEQ_CHECK))
    # ov = 3 with ll = 0 is rep0 - 1: rep0 = 2 gives 1, rep0 = 1 gives 0 (an error), also at the frame's start
    out.append(Case("repeat", "ov3-ll0-rep0=2", [("cmp", skewed(rng, 12), [(10, 4, 2 + 3), (0, 4, 3), (0, 5, 1)])], ov=True))
    out.append(Case("repeat", "ov3-ll0-rep0=1-offset0", [("cmp", skewed(rng, 12), [(10, 4, 1 + 3), (0, 4, 3)])], ov=True,
                    handback=WHY_SEQ_CHECK))
    out.append(Case("repeat", "ov3-ll0-initial-rep0=1-offset0", [("raw", b"abcdefghij"), ("cmp", b"xy", [(0, 4, 3)])], ov=True,
                    handback=WHY_SEQ_CHECK))
    return out


def fse_paths(rng):
    """One sequence with LL code 34 and ML code 51 (15 extra bits each) and a chosen OF code after ~2000 ordinary ones: up to
    FSE_FAST_XBITS extra bits k_fse stays on its fast path, above it the block is replayed by its exact path.  Offset codes
    30 and 31 (offsets beyond any output) go to the exact path and fail."""
    out = []
    for ofcode in (2, 3, 8, 9, 30, 31):
        xbits = 15 + 15 + ofcode
        pre = [(16, 5, 7)] + _ordinary(rng, 1999, 21, ll_max=2, ml_hi=10, of_max=5000)
        pos = sum(q[0] + q[1] for q in pre)
        wide = (32768 + rng.randrange(8000), 32771 + rng.randrange(8000), (1 << ofcode) - 3)
        seqs = pre + [wide] + _ordinary(rng, 40, pos + wide[0] + wide[1], of_max=5000)
        name = f"xbits{xbits}" + ("-fast=FSE_FAST_XBITS" if xbits == FSE_FAST_XBITS else "") + (f"-ofcode{ofcode}" if ofcode >= 30 else "")
        out.append(Case("fse", name, [_cmp(rng, seqs, tail=3)], handback=None if ofcode < 30 else WHY_SEQ_RECORDS, xbits=xbits))
    return out


GROUPS = {"geometry": geometry, "overlap": overlap, "dense": dense, "earlier": earlier_blocks, "cta-block": cta_edges,
          "repeat": repeats, "fse": fse_paths}


def cases(group=None):
    """The crafted cases (all groups, or one), built from fixed seeds."""
    out = []
    for i, (g, fn) in enumerate(GROUPS.items()):
        if group is None or g == group:
            out += fn(random.Random(0x5EC0 + i))
    return out
