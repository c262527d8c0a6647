"""What libzstd writes across its levels, strategies, windows and block shapes: a fixed matrix of frames built with the system
libzstd (datagen.zstd(), with the prototypes below added), and a census of what those frames contain.

The crafted suites (seqcraft, entcraft, hufring, dictcraft, streamcraft) pin the decoder's edges one feature at a time; this
matrix is real encoder output, where the features come combined and at volume: Treeless literals and Repeat tables chained
through hundreds of blocks, all three repeat codes with and without the LL = 0 shift, Raw and RLE blocks between Compressed ones,
offsets of tens of MiB, blocks on k_fse's exact path, frames that k_exec_cta takes alone, dictionaries, multi-threaded,
rsyncable and flushed streams.

Nothing here imports the library: frames come from libzstd, the census from tests/refwalk.py (headers) and the oracle's trace
(sequences).  Frames are cached under datagen.CACHE, keyed by the libzstd version and each frame's parameters."""
import ctypes as C
import hashlib
import os
import random
from concurrent.futures import ThreadPoolExecutor

import numpy as np

import datagen as G
import refwalk

MiB = 1 << 20

# zstd.h 1.5.5: stable parameters and the experimental ones this matrix uses (ZSTD_c_experimentalParam1, 5, 6 and 13)
P = {"compressionLevel": 100, "windowLog": 101, "minMatch": 105, "enableLongDistanceMatching": 160, "contentSizeFlag": 200,
     "checksumFlag": 201, "dictIDFlag": 202, "nbWorkers": 400, "rsyncable": 500, "literalCompressionMode": 1002,
     "targetCBlockSize": 1003, "useBlockSplitter": 1010}
ZSTD_e_continue, ZSTD_e_flush, ZSTD_e_end = 0, 1, 2
ZSTD_d_windowLogMax = 100
SKIPPABLE_MAGIC = 0x184D2A50

FSE_FAST_XBITS = 38     # k_fse's fast path: most extra bits (LL + ML + OF) in one sequence (tests/seqcraft.py)
LL_BASE = np.array(list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64] + [1 << k for k in range(7, 17)], dtype=np.int64)
LL_BITS = np.array([0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16], dtype=np.int64)
ML_BASE = np.array(list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99] + [(1 << k) + 3 for k in range(7, 17)], dtype=np.int64)
ML_BITS = np.array([0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16], dtype=np.int64)

# the oracle's default window limit (ruzstd's MAXIMUM_ALLOWED_WINDOW_SIZE) and the one frames above it are decoded with
DEFAULT_MAX_WINDOW = 128 * MiB
RAISED_MAX_WINDOW = 512 * MiB


class _Bounds(C.Structure):
    _fields_ = [("error", C.c_size_t), ("lowerBound", C.c_int), ("upperBound", C.c_int)]


class _InBuf(C.Structure):
    _fields_ = [("src", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class _OutBuf(C.Structure):
    _fields_ = [("dst", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class _FParams(C.Structure):
    _fields_ = [("contentSizeFlag", C.c_int), ("checksumFlag", C.c_int), ("noDictIDFlag", C.c_int)]


_zx = None


def zstd():
    """datagen's libzstd with the prototypes for streaming, CDicts, ZDICT training and parameter bounds."""
    global _zx
    if _zx is None:
        z = G.zstd()
        vp, sz = C.c_void_p, C.c_size_t
        z.ZSTD_versionNumber.restype = C.c_uint
        z.ZSTD_cParam_getBounds.restype = _Bounds; z.ZSTD_cParam_getBounds.argtypes = [C.c_int]
        z.ZSTD_getErrorName.restype = C.c_char_p; z.ZSTD_getErrorName.argtypes = [sz]
        z.ZSTD_compressStream2.restype = sz
        z.ZSTD_compressStream2.argtypes = [vp, C.POINTER(_OutBuf), C.POINTER(_InBuf), C.c_int]
        z.ZSTD_createCDict.restype = vp; z.ZSTD_createCDict.argtypes = [vp, sz, C.c_int]
        z.ZSTD_freeCDict.argtypes = [vp]
        z.ZSTD_compress_usingCDict_advanced.restype = sz
        z.ZSTD_compress_usingCDict_advanced.argtypes = [vp, vp, sz, vp, sz, vp, _FParams]
        z.ZDICT_trainFromBuffer.restype = sz; z.ZDICT_trainFromBuffer.argtypes = [vp, sz, vp, vp, C.c_uint]
        z.ZDICT_isError.restype = C.c_uint; z.ZDICT_isError.argtypes = [sz]
        z.ZDICT_getDictID.restype = C.c_uint; z.ZDICT_getDictID.argtypes = [vp, sz]
        _zx = z
    return _zx


def version():
    return int(zstd().ZSTD_versionNumber())


def check_param(name, value):
    """Fails with a clear message if the installed libzstd does not know parameter `name` or refuses `value`."""
    z = zstd()
    b = z.ZSTD_cParam_getBounds(P[name])
    if z.ZSTD_isError(b.error):
        raise RuntimeError(f"libzstd {version()} lacks ZSTD_c_{name} (parameter {P[name]}): "
                           f"{z.ZSTD_getErrorName(b.error).decode()}; the matrix needs libzstd 1.5.5's numbering")
    if not b.lowerBound <= value <= b.upperBound:
        raise RuntimeError(f"libzstd {version()}: ZSTD_c_{name} = {value} is outside [{b.lowerBound}, {b.upperBound}]"
                           + (" (a library built without multi-threading)" if name == "nbWorkers" else ""))


def _u8(b):
    return np.frombuffer(bytes(b), dtype=np.uint8)


# ------------------------------------------------------------------------------------------------------------
# inputs (fixed seeds)
# ------------------------------------------------------------------------------------------------------------
def _rle_input():
    return np.concatenate([G.gen_text(64 << 10, 0x2A7051), np.full(384 << 10, 0x61, np.uint8), G.gen_text(64 << 10, 0x2A7052)])


def _far_input():
    """A random 1 MiB block, ~20 MiB of text, the same block again: offsets of ~21 MiB with 128 KiB matches under LDM."""
    blk = np.random.Generator(np.random.PCG64(0x2A7061)).integers(0, 256, MiB, dtype=np.uint8)
    return np.concatenate([blk, G.c2_text_plain(20 * MiB, 0x2A7062), blk])


def _dense_input():
    """256 random 3-byte tokens drawn i.i.d.: at minMatch 3 an optimal parse is one 3-byte match per token and no literals,
    over 0x7F00 sequences in a 128 KiB block, every one with LL = 0."""
    rng = np.random.Generator(np.random.PCG64(0x2A7071))
    tok = rng.integers(0, 256, (256, 3), dtype=np.uint8)
    return tok[rng.integers(0, 256, MiB // 3)].reshape(-1)


def _zins(x, every):
    """`x` with a "z" inserted after every `every` bytes."""
    return np.concatenate([np.concatenate([x[i:i + every], np.frombuffer(b"z", np.uint8)]) for i in range(0, len(x), every)])


def _rlelits_input():
    """256 KiB of random bytes, then two copies of it with a "z" every 400 bytes: the copies are matches whose literals are all
    "z", so their blocks carry RLE literals (and RLE tables)."""
    r = np.random.Generator(np.random.PCG64(0x2A7081)).integers(0, 256, 256 << 10, dtype=np.uint8)
    return np.concatenate([r, _zins(r, 400), _zins(r, 400)])


def _chain_input():
    """256 KiB blocks of 1 KiB, each the one before with a "z" every 40 bytes: at windowLog 11 every block's literals are 8-31 or
    32+ "z"s, RLE literals with 1- and 2-byte headers."""
    ys = [np.random.Generator(np.random.PCG64(0x2A7082)).integers(0, 256, 1024, dtype=np.uint8)]
    for _ in range(255):
        ys.append(_zins(ys[-1], 40)[:1024])
    return np.concatenate(ys)


def _tagged_input():
    """40,000 records of 8 random bytes and a fixed 16-byte tag: every match is the tag, one ML code (ML RLE tables)."""
    rng = np.random.Generator(np.random.PCG64(0x2A7083))
    tag = rng.integers(0, 256, 16, dtype=np.uint8)
    return np.concatenate([rng.integers(0, 256, (40000, 8), dtype=np.uint8), np.tile(tag, (40000, 1))], axis=1).reshape(-1)


INPUTS = {
    "text": lambda: G.c2_text_plain(8 * MiB, 0x2A7001),
    "silesia": lambda: G.gen_silesia_mix(8 * MiB, 0x2A7002),
    "records": lambda: G.gen_binary_records(2 * MiB, 0x2A7003),
    "skewed": lambda: G.gen_skewed_bytes(2 * MiB, 0x2A7004),
    "rle": _rle_input,
    "random": lambda: np.random.Generator(np.random.PCG64(0x2A7005)).integers(0, 256, MiB, dtype=np.uint8),
    "far": _far_input,
    "dense": _dense_input,
    "rlelits": _rlelits_input,
    "chain": _chain_input,
    "tagged": _tagged_input,
}
_inputs = {}


def plain_input(name):
    if name not in _inputs:
        _inputs[name] = INPUTS[name]().tobytes()
    return _inputs[name]


# ------------------------------------------------------------------------------------------------------------
# the matrix
# ------------------------------------------------------------------------------------------------------------
RECIPE = 2   # part of every cache key: change it when inputs or the way frames are written change
LEVELS = (-7, -1, 1, 2, 3, 5, 7, 9, 12, 16, 19, 22)


class Spec:
    """One frame to build: id (what it aims at), input name and length, libzstd parameters, and how it is written:
    "once" (ZSTD_compress2), "flush" (ZSTD_compressStream2 with ZSTD_e_flush every 4-64 KiB), "stream" (one ZSTD_e_end on an
    unknown size), "cdict" (ZSTD_compress_usingCDict_advanced on the trained dictionary) or "rawdict" (ZSTD_compress_usingDict on
    raw content)."""

    def __init__(self, id, input, size, params, how="once", dict_id_flag=True, offset=0):
        self.id, self.input, self.size, self.params, self.how = id, input, size, dict(params), how
        self.dict_id_flag, self.offset = dict_id_flag, offset

    def key(self):
        return repr((version(), RECIPE, self.id, self.input, self.size, self.offset, sorted(self.params.items()), self.how, self.dict_id_flag))

    def plain(self):
        return plain_input(self.input)[self.offset:self.offset + self.size]


def specs():
    L = "compressionLevel"
    out = []
    for lv in LEVELS:
        out.append(Spec(f"level{lv}-silesia", "silesia", 2 * MiB, {L: lv}))
        out.append(Spec(f"level{lv}-text", "text", MiB, {L: lv}))
    out += [
        Spec("wlog10-text-1KiB-blocks", "text", MiB, {L: 3, "windowLog": 10}),
        Spec("wlog17-silesia", "silesia", 8 * MiB, {L: 3, "windowLog": 17}),
        Spec("wlog23-level19-silesia", "silesia", 4 * MiB, {L: 19, "windowLog": 23}),
        Spec("wlog27-ldm-far-offsets", "far", 22 * MiB, {L: 3, "windowLog": 27, "enableLongDistanceMatching": 1}),
        Spec("minmatch3-dense", "dense", MiB, {L: 3, "minMatch": 3}),
        Spec("minmatch3-level19-dense-7f00-seqs", "dense", MiB, {L: 19, "minMatch": 3}),
        Spec("minmatch7-skewed-literals-only", "skewed", MiB, {L: 3, "minMatch": 7}, offset=MiB),
        Spec("minmatch3-records", "records", 2 * MiB, {L: 1, "minMatch": 3}),
        Spec("tcbs1340-text-treeless", "text", 3 * MiB, {L: 3, "targetCBlockSize": 1340}),
        Spec("rawlits-text", "text", MiB, {L: 3, "literalCompressionMode": 2}, offset=MiB),
        Spec("splitter-level9-silesia", "silesia", 4 * MiB, {L: 9, "useBlockSplitter": 1}, offset=2 * MiB),
        Spec("mt4-text", "text", 8 * MiB, {L: 3, "nbWorkers": 4}),
        Spec("mt4-rsyncable-silesia", "silesia", 8 * MiB, {L: 3, "nbWorkers": 4, "rsyncable": 1}),
        Spec("nochecksum-records", "records", 2 * MiB, {L: 3, "checksumFlag": 0}),
        Spec("nofcs-skewed", "skewed", 2 * MiB, {L: 3, "contentSizeFlag": 0}),
        Spec("level3-rle-run", "rle", 512 << 10, {L: 3}),
        Spec("level3-random-raw", "random", MiB, {L: 3}),
        Spec("level19-rle-literals", "rlelits", 788 << 10, {L: 19}),
        Spec("level19-wlog11-rle-literals-1B-header", "chain", 256 << 10, {L: 19, "windowLog": 11}),
        Spec("level19-tagged-ml-rle", "tagged", 960000, {L: 19}),
        Spec("flushed-text-small-blocks", "text", 2 * MiB, {L: 3}, how="flush", offset=3 * MiB),
        Spec("wlog28-stream-256MiB-window", "text", MiB, {L: 3, "windowLog": 28}, how="stream", offset=5 * MiB),
    ]
    for lv in (1, 3, 9, 19):
        for flag in (True, False):
            out.append(Spec(f"cdict-level{lv}" + ("" if flag else "-noid"), "dict", 0, {L: lv}, how="cdict", dict_id_flag=flag))
    for lv in (1, 3, 19):
        out.append(Spec(f"rawdict-level{lv}", "dict", 0, {L: lv}, how="rawdict"))
    return out


# ------------------------------------------------------------------------------------------------------------
# dictionaries
# ------------------------------------------------------------------------------------------------------------
DICT_CAP = 64 << 10
_dicts = {}


def dict_samples():
    """The pieces the dictionary frames compress: 24 text pieces of 1-32 KiB from the training text's vocabulary."""
    rng = random.Random(0x2A7D01)
    t = G.c2_text_plain(2 * MiB, 0x2A7D02).tobytes()
    out = []
    for i in range(24):
        n = rng.randint(1 << 10, 32 << 10)
        o = rng.randint(0, len(t) - n)
        out.append(t[o:o + n])
    return out


def trained_dict():
    """A formatted dictionary from ZDICT_trainFromBuffer on 2 KiB text samples."""
    if "formatted" not in _dicts:
        path = os.path.join(G.CACHE, f"zmatrix_dict_{version()}.bin")
        if os.path.exists(path):
            _dicts["formatted"] = open(path, "rb").read()
        else:
            z = zstd()
            t = G.c2_text_plain(4 * MiB, 0x2A7D03)
            n = 2048
            sizes = np.full(len(t) // n, n, dtype=np.uint64)
            buf = np.empty(DICT_CAP, dtype=np.uint8)
            r = z.ZDICT_trainFromBuffer(buf.ctypes.data, DICT_CAP, t.ctypes.data, sizes.ctypes.data, len(sizes))
            if z.ZDICT_isError(r):
                raise RuntimeError("ZDICT_trainFromBuffer failed")
            _dicts["formatted"] = buf[:r].tobytes()
            _store(path, _dicts["formatted"])
    return _dicts["formatted"]


def trained_dict_id():
    d = trained_dict()
    return int(zstd().ZDICT_getDictID(d, len(d)))


def raw_dict_content():
    """Raw content (no magic number): frames against it carry no dictionary ID and are decoded with it forced."""
    if "raw" not in _dicts:
        _dicts["raw"] = G.c2_text_plain(96 << 10, 0x2A7D04).tobytes()
    return _dicts["raw"]


# ------------------------------------------------------------------------------------------------------------
# building frames
# ------------------------------------------------------------------------------------------------------------
def _check(n, what):
    z = zstd()
    if z.ZSTD_isError(n):
        raise RuntimeError(f"{what}: {z.ZSTD_getErrorName(n).decode()}")
    return n


def _cctx(params):
    """A CCtx with `params`; the content checksum is on unless they turn it off (libzstd's default is off)."""
    z = zstd()
    cctx = z.ZSTD_createCCtx()
    for k, v in {"checksumFlag": 1, **params}.items():
        check_param(k, v)
        _check(z.ZSTD_CCtx_setParameter(cctx, P[k], v), f"ZSTD_c_{k} = {v}")
    return cctx


def _compress_stream(params, data, flush_seed=None):
    """ZSTD_compressStream2 over `data` of unknown size, 64 KiB of input per call (a first call with ZSTD_e_end would tell libzstd
    the size): ZSTD_e_flush after every 4-64 KiB of input (seeded), or none."""
    z = zstd()
    a = _u8(data)
    out = bytearray()
    dst = np.empty(z.ZSTD_compressBound(128 << 10) + (1 << 17), dtype=np.uint8)
    cctx = _cctx(params)
    rng = random.Random(flush_seed)
    try:
        pos = 0
        while True:
            step = rng.randint(4 << 10, 64 << 10) if flush_seed is not None else 64 << 10
            n = min(step, len(a) - pos)
            inb = _InBuf(a.ctypes.data + pos, n, 0)
            op = ZSTD_e_end if pos + n == len(a) else (ZSTD_e_flush if flush_seed is not None else ZSTD_e_continue)
            while True:
                outb = _OutBuf(dst.ctypes.data, len(dst), 0)
                left = _check(z.ZSTD_compressStream2(cctx, C.byref(outb), C.byref(inb), op), "ZSTD_compressStream2")
                out += dst[:outb.pos].tobytes()
                if inb.pos == inb.size and left == 0:
                    break
            pos += n
            if op == ZSTD_e_end:
                return bytes(out)
    finally:
        z.ZSTD_freeCCtx(cctx)


def _build(spec, plain):
    z = zstd()
    a = _u8(plain)
    cap = z.ZSTD_compressBound(len(a))
    dst = np.empty(cap, dtype=np.uint8)
    if spec.how == "flush":
        return _compress_stream(spec.params, plain, flush_seed=0x2A7F)
    if spec.how == "stream":
        return _compress_stream(spec.params, plain)
    if spec.how == "rawdict":
        return G.compress(plain, level=spec.params["compressionLevel"], raw_dict=raw_dict_content())
    cctx = _cctx({} if spec.how == "cdict" else spec.params)
    try:
        if spec.how == "cdict":
            d = trained_dict()
            cd = z.ZSTD_createCDict(d, len(d), spec.params["compressionLevel"])
            try:
                n = z.ZSTD_compress_usingCDict_advanced(cctx, dst.ctypes.data, cap, a.ctypes.data, len(a), cd,
                                                        _FParams(1, 1, 0 if spec.dict_id_flag else 1))
            finally:
                z.ZSTD_freeCDict(cd)
        else:
            n = z.ZSTD_compress2(cctx, dst.ctypes.data, cap, a.ctypes.data, len(a))
        _check(n, spec.id)
    finally:
        z.ZSTD_freeCCtx(cctx)
    return dst[:n].tobytes()


class Frame:
    """A built frame: `data` decodes to `plain`.  dict: None, "formatted" (trained_dict(); `dict_id` False when the frame does not
    name it) or "raw" (raw_dict_content(), no ID).  checksum: written with a content checksum.  max_window: the window limit a
    decoder needs for it (None: the default)."""

    def __init__(self, id, data, plain, dict=None, dict_id=False, checksum=True):
        self.id, self.data, self.plain, self.dict, self.dict_id, self.checksum = id, data, plain, dict, dict_id, checksum
        window = refwalk.frame_header(data)[1]
        self.window = window
        self.max_window = RAISED_MAX_WINDOW if window > DEFAULT_MAX_WINDOW else None

    def __repr__(self):
        return f"Frame({self.id}, {len(self.data)} -> {len(self.plain)})"


def _store(path, data):
    os.makedirs(G.CACHE, exist_ok=True)
    tmp = f"{path}.{os.getpid()}.tmp"
    with open(tmp, "wb") as f:
        f.write(data)
    os.replace(tmp, path)


def _frame_for(spec, fid, plain):
    path = os.path.join(G.CACHE, "zmatrix_" + hashlib.sha256((spec.key() + fid).encode()).hexdigest()[:24] + ".zst")
    if os.path.exists(path):
        data = open(path, "rb").read()
    else:
        data = _build(spec, plain)
        _store(path, data)
    return data


_frames = None


def frames():
    """Every frame of the matrix, in specs() order; built once per process (in a thread pool: ctypes releases the GIL) and cached
    on disk."""
    global _frames
    if _frames is None:
        ss = specs()
        for name in INPUTS:
            plain_input(name)
        trained_dict()
        pieces = dict_samples()
        jobs = []
        for s in ss:
            if s.input == "dict":
                for k, p in enumerate(pieces):
                    jobs.append((s, f"{s.id}/{k}", p))
            else:
                jobs.append((s, s.id, s.plain()))
        # the slowest first, so the pool does not end on one long level-19/22 frame
        order = sorted(range(len(jobs)), key=lambda i: -len(jobs[i][2]) * max(1, jobs[i][0].params.get("compressionLevel", 3)))
        with ThreadPoolExecutor(max_workers=G.nthreads()) as ex:
            built = dict(zip(order, ex.map(lambda i: _frame_for(*jobs[i]), order)))
        out = []
        for i, (s, fid, p) in enumerate(jobs):
            kind = {"cdict": "formatted", "rawdict": "raw"}.get(s.how)
            # ZSTD_compress_usingDict writes no checksum; everything else has one unless the spec turns it off
            out.append(Frame(fid, built[i], p, kind, kind == "formatted" and s.dict_id_flag,
                             s.how != "rawdict" and s.params.get("checksumFlag", 1) == 1))
        _frames = out
    return _frames


def by_id(fs):
    return {f.id: f for f in fs}


# ------------------------------------------------------------------------------------------------------------
# multi-frame buffers
# ------------------------------------------------------------------------------------------------------------
def skippable(payload):
    return SKIPPABLE_MAGIC.to_bytes(4, "little") + len(payload).to_bytes(4, "little") + payload


PZSTD_IDS = [f"level{lv}-text" for lv in LEVELS] + ["level3-rle-run"]
CONCAT_IDS = ["nochecksum-records", "nofcs-skewed", "level3-random-raw", "flushed-text-small-blocks", "wlog10-text-1KiB-blocks",
              "minmatch3-dense", "tcbs1340-text-treeless"]


def multi_frame_buffers(fs):
    """{name: (buffer, plaintext, frame ids)}: pzstd's layout (a 4-byte skippable frame holding the next frame's compressed size in
    front of each frame) and a plain concatenation."""
    b = by_id(fs)
    pz = b"".join(skippable(len(b[i].data).to_bytes(4, "little")) + b[i].data for i in PZSTD_IDS)
    cat = b"".join(b[i].data for i in CONCAT_IDS)
    return {"pzstd": (pz, b"".join(b[i].plain for i in PZSTD_IDS), PZSTD_IDS),
            "concat": (cat, b"".join(b[i].plain for i in CONCAT_IDS), CONCAT_IDS)}


# ------------------------------------------------------------------------------------------------------------
# the oracle's view
# ------------------------------------------------------------------------------------------------------------
def setup_decoder(d, frame, max_window=None):
    """Sets up a FrameDecoder -- the oracle's or the library's, they share the surface -- for `frame`'s dictionary and window and
    resets it on the frame.  Returns the reader."""
    mw = max_window if max_window is not None else frame.max_window
    if mw:
        d.set_max_window_size(mw)
    if frame.dict == "formatted":
        d.add_dict(trained_dict())
    r = d.reset(frame.data)
    if frame.dict == "formatted" and not frame.dict_id:
        d.force_dict(trained_dict_id())
    elif frame.dict == "raw":
        d.add_raw_content_dict(1, raw_dict_content())
        d.force_dict(1)
    return r


def oracle_decoder(oracle, frame, max_window=None):
    """An oracle FrameDecoder set up for `frame` and reset on it: (decoder, reader)."""
    d = oracle.FrameDecoder()
    return d, setup_decoder(d, frame, max_window)


def trace(oracle, frame):
    """The oracle's decode of `frame` with its trace: (plaintext, decoder, blocks, literals, sequences)."""
    d, r = oracle_decoder(oracle, frame)
    d.trace_enable()
    d.decode_blocks(r, oracle.ALL)
    out = d.collect()
    blocks, lits, seqs = d.trace()
    return out, d, blocks, lits, seqs


def exact_path_blocks(blocks, seqs):
    """Per block of the trace: True where k_fse's fast path gives it up for the exact path -- a sequence with more than
    FSE_FAST_XBITS extra bits (LL + ML + OF) or with offset code >= 30 (seqcraft's rule, k_fse's `flags`)."""
    out = []
    for tb in blocks:
        n = tb["num_sequences"] if tb["block_type"] == 2 else 0
        if not n:
            out.append(False)
            continue
        s = seqs[tb["seq_offset"]:tb["seq_offset"] + n].astype(np.int64)
        llb = LL_BITS[np.searchsorted(LL_BASE, s[:, 0], side="right") - 1]
        mlb = ML_BITS[np.searchsorted(ML_BASE, s[:, 1], side="right") - 1]
        ofc = np.floor(np.log2(np.maximum(s[:, 2], 1))).astype(np.int64)
        out.append(bool(((llb + mlb + ofc) > FSE_FAST_XBITS).any() or (ofc >= 30).any()))
    return out


def headers(data):
    """Frame and block headers: (frame facts, [block facts]) from refwalk's restatement of the reference's parsers."""
    desc = data[4]
    pos, window, chk = refwalk.frame_header(data)
    fr = {"single_segment": bool((desc >> 5) & 1), "fcs": bool((desc >> 6) or ((desc >> 5) & 1)), "checksum": bool(chk),
          "dict_id": bool(desc & 3), "window": window}
    blocks = []
    while True:
        bh = int.from_bytes(data[pos:pos + 3], "little"); pos += 3
        last, bt, size = bh & 1, (bh >> 1) & 3, bh >> 3
        b = {"type": bt}
        if bt == 2:
            c = data[pos:pos + size]
            lt, regen, comp, streams, n, payload = refwalk.literals_header(c)
            s = c[n + payload:]
            nseq, modes = refwalk.sequences_header(s)
            b.update(lit_type=lt, lit_header=n, streams=streams, nseq=nseq,
                     seq_format=0 if s[0] == 0 else 1 if s[0] < 128 else 2 if s[0] < 255 else 3,
                     modes=((modes >> 6) & 3, (modes >> 4) & 3, (modes >> 2) & 3) if nseq else None)
        blocks.append(b)
        pos += 1 if bt == 1 else size
        if last:
            return fr, blocks


LIT_TYPES = ("Raw", "RLE", "Compressed", "Treeless")
BLOCK_TYPES = ("Raw", "RLE", "Compressed")
MODES = ("Predefined", "RLE", "FSE", "Repeat")


def census(oracle, fs):
    """Counts what the frames contain (see FLOOR).  Also returns, per frame id, the exact-path flag of each block."""
    from collections import Counter
    c = Counter()
    exact = {}
    largest_offset, blocks_per_frame = 0, []
    for f in fs:
        fr, hb = headers(f.data)
        out, d, blocks, lits, seqs = trace(oracle, f)
        assert out == f.plain, f.id
        assert len(blocks) == len(hb), f.id
        c[f"window_log {int(fr['window']).bit_length() - 1}" if not fr["single_segment"] else "single_segment"] += 1
        for k in ("fcs", "checksum", "dict_id"):
            c[f"frame {'with' if fr[k] else 'without'} {k}"] += 1
        blocks_per_frame.append(len(hb))
        ex = exact_path_blocks(blocks, seqs)
        exact[f.id] = ex
        for b, tb, e in zip(hb, blocks, ex):
            c[f"block {BLOCK_TYPES[b['type']]}"] += 1
            if b["type"] != 2:
                continue
            lt = LIT_TYPES[b["lit_type"]]
            assert b["lit_type"] == tb["literals_type"] and b["nseq"] == tb["num_sequences"], f.id
            c[f"literals {lt}"] += 1
            c[f"literals {lt} header {b['lit_header']}B"] += 1
            if b["lit_type"] >= 2:
                c[f"literals {b['streams']} stream(s)"] += 1
            c[f"nseq format {b['seq_format']}B" if b["nseq"] else "nseq format 0"] += 1
            if b["modes"]:
                for kind, m in zip(("LL", "OF", "ML"), b["modes"]):
                    c[f"{kind} {MODES[m]}"] += 1
                c["modes LL/OF/ML " + "/".join(MODES[m] for m in b["modes"])] += 1
            c["exact-path blocks"] += e
            if b["nseq"]:
                s = seqs[tb["seq_offset"]:tb["seq_offset"] + b["nseq"]].astype(np.int64)
                for ov in (1, 2, 3):
                    sel = s[:, 2] == ov
                    c[f"Offset_Value {ov} LL>0"] += int((sel & (s[:, 0] > 0)).sum())
                    c[f"Offset_Value {ov} LL=0"] += int((sel & (s[:, 0] == 0)).sum())
                mo = int(s[:, 3].max())
                largest_offset = max(largest_offset, mo)
                for lg in (17, 23, 24):
                    c[f"offsets > 2^{lg}"] += int((s[:, 3] > (1 << lg)).sum())
                for code in np.unique(np.floor(np.log2(s[:, 2])).astype(np.int64)):
                    c[f"OF code {int(code)}"] += 1
    c["largest offset"] = largest_offset
    c["most blocks in a frame"] = max(blocks_per_frame)
    c["frames of 500+ blocks"] = sum(1 for n in blocks_per_frame if n >= 500)
    c["frames"] = len(fs)
    return c, exact


# The floor the census must meet, item by item.  A value is the least count; UNREACHABLE names an item libzstd does not write
# and the crafted case that covers it instead.
FLOOR = {**{f"block {t}": 1 for t in BLOCK_TYPES},
         **{f"literals {t}": 1 for t in LIT_TYPES},
         "literals Raw header 1B": 1, "literals Raw header 2B": 1, "literals Raw header 3B": 1,
         "literals RLE header 1B": 1,
         "literals Compressed header 3B": 1, "literals Compressed header 4B": 1, "literals Compressed header 5B": 1,
         "literals Treeless header 3B": 1, "literals Treeless header 4B": 1, "literals Treeless header 5B": 1,
         "literals 1 stream(s)": 1, "literals 4 stream(s)": 1,
         "nseq format 0": 1, "nseq format 1B": 1, "nseq format 2B": 1, "nseq format 3B": 1,
         **{f"{k} {m}": 1 for k in ("LL", "OF", "ML") for m in MODES},
         **{f"Offset_Value {v} LL{s}": 1 for v in (1, 2, 3) for s in (">0", "=0")},
         "offsets > 2^17": 1, "offsets > 2^23": 1, "offsets > 2^24": 1,
         "exact-path blocks": 1, "frames of 500+ blocks": 1,
         **{f"frame {w} {k}": 1 for w in ("with", "without") for k in ("fcs", "checksum", "dict_id")}}
UNREACHABLE = {}


def format_census(c):
    keys = sorted(c, key=lambda k: (k.split()[0], k))
    w = max(len(k) for k in keys)
    return "\n".join(f"| {k:<{w}} | {c[k]:>12,} |" for k in keys)
