"""The batch compressor against a dictionary, on the GPU: every frame must decode with libzstd, with the oracle (ruzstd's decode
semantics) and with this library's decoders given the same dictionary, carry the right dictionary ID (none for raw content) and
checksum, stay within compress_bound_dict and the 128 KiB window, and actually use the dictionary."""
import struct

import numpy as np
import pytest

import datagen
from conftest import read_golden

pytestmark = pytest.mark.gpu

WINDOW = 131072
ENC_MIN_MATCH = 5


@pytest.fixture(scope="module")
def c5():
    """The first 2,000 frames of C5 (1-8 KiB pieces drawn mostly from a 112,640-byte raw-content dictionary) and the dictionary."""
    fs = datagen.config_c5(nframes=2000, cache=False)
    plain = fs.plain.tobytes()
    pieces = [plain[int(o):int(o + n)] for o, n in zip(fs.out_off, fs.out_size)]
    return pieces, fs.raw_dict.tobytes()


def compress_many(pkg, ctx, datas, dict=None, level=1, checksum=True, device=False):
    io = np.zeros(len(datas), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    so = oo = 0
    for i, d in enumerate(datas):
        cap = pkg.compress_bound(len(d), dict)
        io[i] = (so, len(d), oo, cap)
        so += len(d)
        oo += cap
    src = np.frombuffer(b"".join(datas), dtype=np.uint8) if so else np.zeros(1, dtype=np.uint8)
    out = np.zeros(max(oo, 1), dtype=np.uint8)
    if device:
        import torch
        src_t, out_t = torch.from_numpy(src.copy()).cuda(), torch.zeros(out.size, dtype=torch.uint8, device="cuda")
        res = pkg.compress_frames(ctx, src_t, io, out_t, level, checksum, dict=dict)
        out = out_t.cpu().numpy()
    else:
        res = pkg.compress_frames(ctx, src, io, out, level, checksum, dict=dict)
    frames = []
    for i in range(len(datas)):
        assert res[i]["status"] == 0
        frames.append(out[io[i]["dst_off"]:io[i]["dst_off"] + res[i]["dst_size"]].tobytes())
    return frames, res


def old_entry(pkg, ctx, datas):
    """The frames b200z_compress_frames_batch (the entry without a dictionary argument) writes."""
    io = np.zeros(len(datas), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    so = oo = 0
    for i, d in enumerate(datas):
        cap = pkg.compress_bound(len(d))
        io[i] = (so, len(d), oo, cap)
        so += len(d)
        oo += cap
    src = np.frombuffer(b"".join(datas), dtype=np.uint8) if so else np.zeros(1, dtype=np.uint8)
    out = np.zeros(max(oo, 1), dtype=np.uint8)
    res = np.zeros(len(io), dtype=pkg.binding.COMPRESS_RESULT_DTYPE)
    assert pkg.lib().b200z_compress_frames_batch(ctx.h, src.ctypes.data, src.size, 0, io.ctypes.data, len(io), 1, 1, out.ctypes.data, out.size, 0,
                                                 res.ctypes.data) == 0
    return [out[io[i]["dst_off"]:io[i]["dst_off"] + res[i]["dst_size"]].tobytes() for i in range(len(datas))]


def header_dict_id(f):
    """(has a dictionary ID field, the ID) from a frame header."""
    n = (0, 1, 2, 4)[f[4] & 3]
    return n > 0, int.from_bytes(f[6:6 + n], "little")


def oracle_trace(oracle, f, content=None, formatted=None):
    """Decodes f with the oracle (raw content forced, or a formatted dictionary by ID); returns (output, sequences whose source lies
    before the frame's first byte, largest offset).  Checks the declared window, each block's size, and that a source in the
    dictionary stops at the dictionary's end (the compressor does not run a match from the dictionary into the frame)."""
    d = oracle.FrameDecoder()
    d.trace_enable()
    if formatted is not None:
        d.add_dict(formatted)
    if content is not None:
        d.add_raw_content_dict(1, content)
    r = d.reset(f)
    if content is not None:
        d.force_dict(1)
    d.decode_blocks(r)
    out = d.collect()
    blocks, _, seqs = d.trace()
    assert d.window_size() == WINDOW
    assert all(b["out_size"] <= WINDOW for b in blocks)
    before = 0
    for b in blocks:
        pos, k = int(b["out_offset"]), int(b["seq_offset"])
        for ll, ml, _, off in seqs[k:k + int(b["num_sequences"])].tolist():
            pos += ll
            before += off > pos
            assert off <= pos or off - pos >= ml, (pos, ll, ml, off)
            pos += ml
    return out, before, int(seqs[:, 3].max()) if len(seqs) else 0


def oracle_trace_seqs(oracle, f, content):
    d = oracle.FrameDecoder()
    d.trace_enable()
    d.add_raw_content_dict(1, content)
    r = d.reset(f)
    d.force_dict(1)
    d.decode_blocks(r)
    d.collect()
    return d.trace()


def batch_decode(pkg, ctx, datas, frames, dicts=None, forced=None):
    io = np.zeros(len(frames), dtype=pkg.binding.FRAME_IO_DTYPE)
    so = oo = 0
    for i, (f, d) in enumerate(zip(frames, datas)):
        io[i] = (so, len(f), oo, len(d))
        so += len(f)
        oo += len(d)
    out = np.zeros(oo + 16, dtype=np.uint8)
    res = pkg.decode_frames(ctx, np.frombuffer(b"".join(frames), dtype=np.uint8), io, out, dicts=dicts, forced_dict=forced)
    for i, d in enumerate(datas):
        assert res[i]["status"] == 0 and res[i]["out_size"] == len(d), i
        assert out[io[i]["out_off"]:io[i]["out_off"] + len(d)].tobytes() == d, i


def check_raw_content(pkg, ctx, oracle, D, content, datas, frames, res, monkeypatch):
    """Every check of a raw-content round trip; returns the number of sequences that reach into the dictionary."""
    before = 0
    for d, f, r in zip(datas, frames, res):
        assert len(f) <= pkg.compress_bound(len(d), D)
        assert header_dict_id(f) == (False, 0)
        assert datagen.decompress(f, len(d), raw_dict=content) == d
        out, b, max_off = oracle_trace(oracle, f, content=content)
        assert out == d and max_off <= WINDOW
        before += b
        want = pkg.xxh64(d) & 0xFFFFFFFF
        assert r["has_checksum"] == 1 and r["checksum"] == want and struct.unpack("<I", f[-4:])[0] == want
    for mode in ("warp", "cta"):
        monkeypatch.setenv("B200Z_EXEC_MODE", mode)
        batch_decode(pkg, ctx, datas, frames, forced=D)
    monkeypatch.delenv("B200Z_EXEC_MODE")
    dec = pkg.FrameDecoder(ctx)
    dec.add_raw_content_dict(1, content)
    for d, f in zip(datas, frames):
        r = dec.reset(f)
        dec.force_dict(1)
        dec.decode_blocks(r, pkg.ALL)
        assert dec.collect() == d
    return before


def boundary_frames(content):
    """A match ending exactly at the dictionary's end, and a source that runs from the dictionary into the frame."""
    t = content[-64:]
    other = bytes(np.random.default_rng(7).integers(0, 256, 300, dtype=np.uint8))
    return [t + other, t + t + other]


def test_raw_content_round_trip(pkg, ctx, oracle, c5, monkeypatch):
    pieces, content = c5
    D = pkg.Dictionary.raw_content(ctx, 1, content)
    extra = [bytes(datagen.gen_text(n, 31 + n)) if n else b"" for n in (0, 1, 5, 131071, 131073)]
    extra += [b"\x2a" * (300 << 10), np.random.default_rng(5).integers(0, 256, 1 << 20, dtype=np.uint8).tobytes(),
              bytes(datagen.gen_text((8 << 20) + 7, 32))]
    datas = pieces + extra + boundary_frames(content)
    frames, res = compress_many(pkg, ctx, datas, dict=D)
    before = check_raw_content(pkg, ctx, oracle, D, content, datas, frames, res, monkeypatch)
    assert before > len(pieces)   # the C5 pieces are mostly dictionary text
    for f in frames[-2:]:   # both start with a match into the dictionary's last 64 bytes (oracle_trace: it stops at the end)
        _, _, seqs = oracle_trace_seqs(oracle, f, content)
        assert seqs[0][0] == 0 and seqs[0][1] >= ENC_MIN_MATCH and seqs[0][3] <= 64, seqs[:3]


def test_device_resident_and_to_vec(pkg, ctx, oracle, c5):
    pieces, content = c5
    D = pkg.Dictionary.raw_content(ctx, 1, content)
    datas = pieces[:50]
    host, _ = compress_many(pkg, ctx, datas, dict=D)
    dev, _ = compress_many(pkg, ctx, datas, dict=D, device=True)
    assert host == dev
    assert pkg.compress_to_vec(ctx, datas[3], dict=D) == host[3]
    plain = pkg.compress_to_vec(ctx, datas[3], checksum=False, dict=D)
    assert datagen.decompress(plain, len(datas[3]), raw_dict=content) == datas[3]


def test_formatted_round_trip(pkg, ctx, oracle, manifest):
    dic = read_golden("dict_tests", "dictionary")
    names = sorted(manifest["dict"])
    datas = [oracle.decode_frame(read_golden("dict_tests", "files", n), dict_raw=dic)[0] for n in names]
    D = pkg.Dictionary.decode_dict(ctx, dic)
    frames, res = compress_many(pkg, ctx, datas, dict=D)
    for d, f, r in zip(datas, frames, res):
        assert len(f) <= pkg.compress_bound(len(d), D)
        assert header_dict_id(f) == (True, D.id)
        out, _, max_off = oracle_trace(oracle, f, formatted=dic)
        assert out == d and max_off <= WINDOW
        assert datagen.decompress(f, len(d), raw_dict=dic) == d
        assert r["checksum"] == pkg.xxh64(d) & 0xFFFFFFFF
    batch_decode(pkg, ctx, datas, frames, dicts=[D])


def test_dictionary_used_within_window(pkg, ctx, oracle):
    """A 1 MiB dictionary: frames drawn from all over it reach back into it, but never further than the window."""
    content = bytes(datagen.gen_text(1 << 20, 41))
    rng = np.random.default_rng(9)
    datas = []
    for _ in range(64):
        parts = []
        for _ in range(12):
            o = int(rng.integers(0, len(content) - 512))
            parts.append(content[o:o + 300])
        datas.append(b"".join(parts))
    D = pkg.Dictionary.raw_content(ctx, 1, content)
    frames, _ = compress_many(pkg, ctx, datas, dict=D)
    before = 0
    for d, f in zip(datas, frames):
        out, b, max_off = oracle_trace(oracle, f, content=content)
        assert out == d and max_off <= WINDOW
        assert datagen.decompress(f, len(d), raw_dict=content) == d
        before += b
    assert before > 0


def test_window_sized_dictionary_boundary(pkg, ctx, oracle, monkeypatch):
    """A 131,072-byte dictionary and a frame of that dictionary then 4 KiB of it again: position 0 may match dictionary byte 0 at
    offset 131,072 exactly, and no offset goes beyond it."""
    content = bytes(datagen.gen_text(WINDOW, 51))
    D = pkg.Dictionary.raw_content(ctx, 1, content)
    datas = [content + content[:4096]]
    frames, res = compress_many(pkg, ctx, datas, dict=D)
    check_raw_content(pkg, ctx, oracle, D, content, datas, frames, res, monkeypatch)
    _, before, max_off = oracle_trace(oracle, frames[0], content=content)
    assert before > 0 and max_off <= WINDOW
    print(f"window-sized dictionary: largest offset {max_off}, {before} sequences into the dictionary")


def test_ratio_floor_on_c5_frames(pkg, ctx, c5):
    pieces, content = c5
    D = pkg.Dictionary.raw_content(ctx, 1, content)
    total = sum(len(p) for p in pieces)
    with_dict = total / sum(len(f) for f in compress_many(pkg, ctx, pieces, dict=D, checksum=False)[0])
    without = total / sum(len(f) for f in compress_many(pkg, ctx, pieces, checksum=False)[0])
    zstd1 = total / sum(len(datagen.compress(p, level=1, raw_dict=content)) for p in pieces)
    print(f"ratio on 2,000 C5 frames (no checksum): with the dictionary {with_dict:.3f}, without {without:.3f}, "
          f"libzstd level 1 with the dictionary {zstd1:.3f}")
    assert with_dict >= 0.8 * zstd1
    assert with_dict >= 1.75 * without


def test_null_and_empty_dictionaries(pkg, ctx, manifest, oracle):
    from test_compress import _inputs
    ins = _inputs(manifest, oracle)
    datas = [ins[n] for n in sorted(ins)]
    old = old_entry(pkg, ctx, datas)
    assert compress_many(pkg, ctx, datas)[0] == old
    E = pkg.Dictionary.raw_content(ctx, 1, b"")
    assert compress_many(pkg, ctx, datas, dict=E)[0] == old
    assert pkg.compress_bound(1000, E) == pkg.compress_bound(1000)


def test_deterministic(pkg, ctx, c5):
    pieces, content = c5
    D = pkg.Dictionary.raw_content(ctx, 1, content)
    a = pieces[:300]
    f1, _ = compress_many(pkg, ctx, a, dict=D)
    f2, _ = compress_many(pkg, ctx, a, dict=D)
    assert f1 == f2
    f3, _ = compress_many(pkg, ctx, [pieces[500], a[17], bytes(datagen.gen_text(200000, 61)), a[250]], dict=D)
    assert f3[1] == f1[17] and f3[3] == f1[250]
    del D
    launches = ctx.kernel_launches()
    D2 = pkg.Dictionary.raw_content(ctx, 1, content)
    f4, _ = compress_many(pkg, ctx, a, dict=D2)
    assert f4 == f1
    assert ctx.kernel_launches() - launches == 5   # k_cdict once, then the four stages
    compress_many(pkg, ctx, a, dict=D2)
    assert ctx.kernel_launches() - launches == 9


def test_uncompressed_level_with_dictionary(pkg, ctx, manifest):
    dic = read_golden("dict_tests", "dictionary")
    D = pkg.Dictionary.decode_dict(ctx, dic)
    d = bytes(datagen.gen_text(1000, 71))
    f = pkg.compress_to_vec(ctx, d, level=pkg.UNCOMPRESSED, dict=D)
    want = struct.pack("<IBBI", 0xFD2FB528, (1 << 6) | 4 | 3, 7 << 3, D.id) + struct.pack("<H", 1000 - 256)
    want += struct.pack("<I", 1 | (1000 << 3))[:3] + d + struct.pack("<I", pkg.xxh64(d) & 0xFFFFFFFF)
    assert f == want and len(f) <= pkg.compress_bound(1000, D)


def test_rejections_before_any_launch(pkg, ctx):
    L = pkg.lib()
    err = {v: k for k, v in pkg.error_names().items()}
    dic = read_golden("dict_tests", "dictionary")
    D = pkg.Dictionary.decode_dict(ctx, dic)
    R = pkg.Dictionary.raw_content(ctx, 1, bytes(datagen.gen_text(4096, 81)))
    other = pkg.Context(0)
    X = pkg.Dictionary.raw_content(other, 1, bytes(datagen.gen_text(4096, 81)))
    src = np.zeros(1000, dtype=np.uint8)
    out = np.zeros(4096, dtype=np.uint8)
    assert pkg.compress_bound(1000, D) == pkg.compress_bound(1000) + 4 and pkg.compress_bound(1000, R) == pkg.compress_bound(1000)

    def call(rows, dict, level=1):
        io = np.array(rows, dtype=pkg.binding.COMPRESS_IO_DTYPE)
        res = np.zeros(len(io), dtype=pkg.binding.COMPRESS_RESULT_DTYPE)
        return L.b200z_compress_frames_batch_dict(ctx.h, src.ctypes.data, src.size, 0, io.ctypes.data, len(io), level, 1, dict.h,
                                                  out.ctypes.data, out.size, 0, res.ctypes.data)

    before = ctx.kernel_launches()
    for d in (D, R):
        bound = pkg.compress_bound(1000, d)
        assert call([(0, 1000, 0, bound - 1)], d) == err["B200Z_ERR_INVALID_ARGUMENT"]
        assert call([(0, 1000, 0, bound)], d, level=9) == err["B200Z_ERR_INVALID_ARGUMENT"]
        for level in (2, 3, 4):
            assert call([(0, 1000, 0, bound)], d, level=level) == err["B200Z_ERR_REFERENCE_WOULD_PANIC"]
    assert call([(0, 1000, 0, pkg.compress_bound(1000))], X) == err["B200Z_ERR_INVALID_ARGUMENT"]
    assert ctx.kernel_launches() == before
    assert call([(0, 1000, 0, pkg.compress_bound(1000, D))], D) == 0
    del X
    other.close()
