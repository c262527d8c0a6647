"""The dictionary finalizer on the GPU (b200z_dict_finalize): its statistics are exactly those of the compressor's parse against the
content (rebuilt on the CPU from the oracle's trace of the compressor's frames), across several statistics submissions, for samples
in host or device memory and on two contexts; the dictionaries it writes load in this library, the oracle and libzstd, and this
library's compressor uses them (frames carry their ID and decode everywhere); bad arguments are refused before any launch."""
import bisect
import ctypes as C
import struct

import numpy as np
import pytest

import datagen
from test_compress_dict import batch_decode, compress_many, header_dict_id

pytestmark = pytest.mark.gpu

LIT, LL, ML, OF = 0, 256, 256 + 36, 256 + 36 + 53
NBINS = OF + 32
DS_BLOCKS = 2048   # samples per statistics submission (csrc/compress.h)
# code baselines of RFC 8878 section 3.1.1.3.2.1.1: a value's code is the last one whose baseline does not exceed it
LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64] + [1 << k for k in range(7, 17)]
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99] + [(1 << k) + 3 for k in range(7, 17)]


@pytest.fixture(scope="module")
def c5():
    """C5 frames 0-3999 (1-8 KiB pieces drawn mostly from a 112,640-byte content) and that content."""
    fs = datagen.config_c5(nframes=4000, cache=False)
    plain = fs.plain.tobytes()
    return [plain[int(o):int(o + n)] for o, n in zip(fs.out_off, fs.out_size)], fs.raw_dict.tobytes()


def counts_from_trace(oracle, frames, content):
    """The statistics of the compressor's first blocks, from the oracle's decode of its frames (raw content forced): literal bytes
    of each block's literals section, LL / ML codes of its sequences and OF codes of their offset values (offset + 3)."""
    cnt = np.zeros(NBINS, dtype=np.uint64)
    for f in frames:
        d = oracle.FrameDecoder()
        d.trace_enable()
        d.add_raw_content_dict(1, content)
        r = d.reset(f)
        d.force_dict(1)
        d.decode_blocks(r)
        d.collect()
        blocks, lits, seqs = d.trace()
        b = blocks[0]
        assert b["block_type"] == 2
        lo = int(b["lit_offset"])
        cnt[LIT:LIT + 256] += np.bincount(np.frombuffer(lits[lo:lo + int(b["regenerated_size"])], dtype=np.uint8), minlength=256).astype(np.uint64)
        k = int(b["seq_offset"])
        for ll, ml, of, _ in seqs[k:k + int(b["num_sequences"])].tolist():
            cnt[LL + bisect.bisect_right(LL_BASE, ll) - 1] += 1
            cnt[ML + bisect.bisect_right(ML_BASE, ml) - 1] += 1
            cnt[OF + of.bit_length() - 1] += 1
    return cnt


def compressed_samples(pkg, ctx, content, candidates):
    """The candidates whose single block the compressor writes as a Compressed block against the raw content, and their frames."""
    D = pkg.Dictionary.raw_content(ctx, 1, content)
    frames, res = compress_many(pkg, ctx, candidates, dict=D, checksum=False)
    keep = [i for i in range(len(candidates)) if res[i]["raw_blocks"] == 0 and res[i]["rle_blocks"] == 0]
    return [candidates[i] for i in keep], [frames[i] for i in keep]


def test_statistics_are_the_compressors_parse(pkg, ctx, oracle, c5):
    import torch
    pieces, content = c5
    plain = b"".join(pieces)
    cand = [plain[i * 1024:(i + 1) * 1024] for i in range(9300)]
    samples, frames = compressed_samples(pkg, ctx, content, cand)
    assert len(samples) > 2 * DS_BLOCKS, len(samples)
    want = pkg.dict_from_counts(counts_from_trace(oracle, frames, content), content)
    before = ctx.kernel_launches()
    got = pkg.finalize_dict(ctx, content, samples)
    nsub = -(-len(samples) // DS_BLOCKS)
    assert ctx.kernel_launches() - before == 1 + 2 * nsub   # k_cdict, then k_cmatch and k_dstats per submission
    assert got == want
    data = b"".join(samples)
    dev = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    assert pkg.finalize_dict(ctx, content, dev, [len(s) for s in samples]) == want
    other = pkg.Context(0)
    try:
        assert pkg.finalize_dict(other, content, data, [len(s) for s in samples]) == want
    finally:
        other.close()


def test_long_samples_count_their_first_block_only(pkg, ctx, oracle, c5):
    """Samples above 128 KiB: only their first 131,072 bytes are parsed (ZDICT_countEStats' rule); RLE samples count nothing."""
    pieces, content = c5
    long1 = b"".join(pieces[:60])
    assert len(long1) > 131072
    samples, frames = compressed_samples(pkg, ctx, content, [long1[:131072], pieces[70], b"", b"a"])
    assert len(samples) == 2
    want = pkg.dict_from_counts(counts_from_trace(oracle, frames, content), content)
    assert pkg.finalize_dict(ctx, content, [long1, pieces[70], b"", b"z" * 5000]) == want


def test_no_samples_gives_the_flat_tables(pkg, ctx, c5):
    _, content = c5
    before = ctx.kernel_launches()
    d = pkg.finalize_dict(ctx, content, [])
    assert ctx.kernel_launches() == before
    assert d == pkg.dict_from_counts(np.zeros(NBINS, dtype=np.uint64), content)


def test_finalized_dictionary_round_trips(pkg, ctx, oracle, c5, monkeypatch):
    """Finalized on C5 0-1999, used on the held-out 2000-3999 and edge inputs: Dictionary.decode_dict parses it, the frames carry
    its ID and decode with libzstd, the oracle (by ID), decode_frames in both execution modes and FrameDecoder.add_dict."""
    pieces, content = c5
    d = pkg.finalize_dict(ctx, content, pieces[:2000])
    did = struct.unpack_from("<I", d, 4)[0]
    D = pkg.Dictionary.decode_dict(ctx, d)
    assert D.id == did >= 32768 and D.offset_hist == [1, 4, 8] and d.endswith(content)
    extra = [bytes(datagen.gen_text(n, 31 + n)) if n else b"" for n in (0, 1, 131071, 131073)]
    extra += [b"\x2a" * 5000, np.random.default_rng(5).integers(0, 256, 100000, dtype=np.uint8).tobytes(), bytes(datagen.gen_text(8 << 20, 32))]
    datas = pieces[2000:] + extra
    frames, res = compress_many(pkg, ctx, datas, dict=D)
    for x, f, r in zip(datas, frames, res):
        assert header_dict_id(f) == (True, did) and len(f) <= pkg.compress_bound(len(x), D)
        assert r["checksum"] == pkg.xxh64(x) & 0xFFFFFFFF and struct.unpack("<I", f[-4:])[0] == r["checksum"]
        assert datagen.decompress(f, len(x), raw_dict=d) == x
        dec = oracle.FrameDecoder()
        dec.add_dict(d)
        rd = dec.reset(f)
        dec.decode_blocks(rd)
        assert dec.collect() == x
    for mode in ("warp", "cta"):
        monkeypatch.setenv("B200Z_EXEC_MODE", mode)
        batch_decode(pkg, ctx, datas, frames, dicts=[D])
    monkeypatch.delenv("B200Z_EXEC_MODE")
    fd = pkg.FrameDecoder(ctx)
    fd.add_dict(d)
    for x, f in zip(datas[::97], frames[::97]):
        r = fd.reset(f)
        fd.decode_blocks(r, pkg.ALL)
        assert fd.collect() == x
    # the same content as raw content: the parse is the same, so the frames differ only by the ID field
    R = pkg.Dictionary.raw_content(ctx, 1, content)
    raw, _ = compress_many(pkg, ctx, pieces[2000:2100], dict=R)
    n = 1 + (did > 0xFFFF) * 2 + (did > 0xFF)
    for a, b in zip(raw, frames[:100]):
        assert b[:4] + bytes([b[4] & ~3]) + b[5:6] + b[6 + n:] == a


def test_create_dict_and_ratio(pkg, ctx, c5):
    pieces, content = c5
    train, held = pieces[:2000], pieces[2000:]
    d = pkg.create_dict(ctx, train, 112640)
    raw = pkg.create_raw_dict(ctx, train, 112640)
    assert len(d) == 112640 and d == pkg.finalize_dict(ctx, raw, train, dict_cap=112640)
    assert d.endswith(raw[-(112640 - 400):])
    assert struct.unpack_from("<I", d, 4)[0] == struct.unpack_from("<I", pkg.create_dict(ctx, train, 112640), 4)[0]
    assert struct.unpack_from("<I", pkg.create_dict(ctx, train, 112640, dict_id=1234), 4)[0] == 1234
    fin = pkg.finalize_dict(ctx, content, train)
    D, R = pkg.Dictionary.decode_dict(ctx, fin), pkg.Dictionary.raw_content(ctx, 1, content)
    total = sum(len(p) for p in held)
    own = total / sum(len(f) for f in compress_many(pkg, ctx, held, dict=D, checksum=False)[0])
    own_raw = total / sum(len(f) for f in compress_many(pkg, ctx, held, dict=R, checksum=False)[0])
    z1 = total / sum(len(datagen.compress(p, level=1, raw_dict=fin)) for p in held)
    z3 = total / sum(len(datagen.compress(p, level=3, raw_dict=fin)) for p in held)
    print(f"held-out C5 ratio: this compressor {own:.3f} with the finalized dictionary ({own_raw:.3f} with its raw content); "
          f"libzstd with it: level 1 {z1:.3f}, level 3 {z3:.3f}")
    # without dict_tables the finalized dictionary only adds its ID field to every frame (test_gpu_dict_tables.py covers the tables)
    assert own_raw * 0.97 <= own <= own_raw


def test_rejections_before_any_launch(pkg, ctx, c5):
    L = pkg.lib()
    bad = {v: k for k, v in pkg.error_names().items()}["B200Z_ERR_INVALID_ARGUMENT"]
    pieces, content = c5
    data = np.frombuffer(b"".join(pieces[:10]), dtype=np.uint8)
    sizes = np.array([len(p) for p in pieces[:10]], dtype=np.uint64)
    out = np.zeros(len(content) + 1000, dtype=np.uint8)
    dlen = C.c_size_t()
    hmax = pkg.binding.DICT_HEADER_MAX

    def call(clen=len(content), sz=sizes, n=data.size, dict_id=0, cap=out.size):
        return L.b200z_dict_finalize(ctx.h, content, clen, data.ctypes.data, n, 0, sz.ctypes.data, len(sz), dict_id, out.ctypes.data, cap,
                                     C.byref(dlen))
    before = ctx.kernel_launches()
    assert call(clen=7) == bad
    assert call(cap=hmax + 7) == bad
    assert call(dict_id=1 << 31) == bad and call(dict_id=0xFFFFFFFF) == bad
    s2 = sizes.copy()
    s2[3] += 1
    assert call(sz=s2) == bad
    s2[3] -= 2
    assert call(sz=s2) == bad
    assert ctx.kernel_launches() == before
    assert call(cap=hmax + 8) == 0 and dlen.value <= hmax + 8
    assert ctx.kernel_launches() == before + 3
    assert call(clen=8, dict_id=(1 << 31) - 1) == 0 and struct.unpack_from("<I", out, 4)[0] == (1 << 31) - 1
