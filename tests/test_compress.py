"""The batch compressor on the GPU: every frame it writes must decode to its input with libzstd, with the oracle (ruzstd's decode
semantics) and with this library's own decoder (batch entry with either execution kernel, and FrameDecoder), carry the right
content checksum and stay within compress_bound."""
import struct

import numpy as np
import pytest

import datagen
from conftest import read_golden

pytestmark = pytest.mark.gpu


def _inputs(manifest, oracle):
    ins = {f"size{n}": datagen.gen_text(n, 11 + n) if n else b"" for n in (0, 1, 5, 131071, 131072, 131073)}
    ins = {k: bytes(v) for k, v in ins.items()}
    ins["rle300k"] = b"\x2a" * (300 << 10)
    ins["random1m"] = np.random.default_rng(3).integers(0, 256, 1 << 20, dtype=np.uint8).tobytes()
    ins["text128k"] = bytes(datagen.gen_text(131072, 21))
    ins["text8m7"] = bytes(datagen.gen_text((8 << 20) + 7, 22))
    ins["silesia"] = bytes(datagen.gen_silesia_mix(3 << 20, 23))
    ins["records"] = bytes(datagen.gen_binary_records(1 << 20, 24))
    ins["skewed"] = bytes(datagen.gen_skewed_bytes(1 << 20, 25))
    for name in sorted(manifest["corpus"]):
        ins["corpus/" + name] = oracle.decode_frame(read_golden("decodecorpus", name))[0]
    return ins


@pytest.fixture(scope="module")
def inputs(manifest, oracle):
    return _inputs(manifest, oracle)


def compress_many(pkg, ctx, datas, level=1, checksum=True, device=False):
    io = np.zeros(len(datas), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    so = oo = 0
    for i, d in enumerate(datas):
        cap = pkg.compress_bound(len(d))
        io[i] = (so, len(d), oo, cap)
        so += len(d)
        oo += cap
    src = np.frombuffer(b"".join(datas), dtype=np.uint8) if so else np.zeros(1, dtype=np.uint8)
    out = np.zeros(max(oo, 1), dtype=np.uint8)
    if device:
        import torch
        src_t, out_t = torch.from_numpy(src.copy()).cuda(), torch.zeros(out.size, dtype=torch.uint8, device="cuda")
        res = pkg.compress_frames(ctx, src_t, io, out_t, level, checksum)
        out = out_t.cpu().numpy()
    else:
        res = pkg.compress_frames(ctx, src, io, out, level, checksum)
    frames = []
    for i in range(len(datas)):
        assert res[i]["status"] == 0
        frames.append(out[io[i]["dst_off"]:io[i]["dst_off"] + res[i]["dst_size"]].tobytes())
    return frames, res


WINDOW = 131072   # the window the compressor's frame headers declare


def within_window(oracle, f):
    """Through the oracle's trace: every block decodes to <= WINDOW bytes and every actual offset is <= WINDOW.  (libzstd's
    one-shot decode and the oracle's offset check against the undrained buffer would both accept an offset beyond it.)"""
    d = oracle.FrameDecoder()
    d.trace_enable()
    r = d.reset(f)
    d.decode_blocks(r)
    out = d.collect()
    blocks, _, seqs = d.trace()
    assert d.window_size() == WINDOW
    assert all(b["out_size"] <= WINDOW for b in blocks)
    assert len(seqs) == 0 or int(seqs[:, 3].max()) <= WINDOW
    return out


def check_frames(pkg, ctx, oracle, datas, frames, res, checksum=True):
    for d, f, r in zip(datas, frames, res):
        assert len(f) <= pkg.compress_bound(len(d))
        assert datagen.decompress(f, len(d)) == d
        assert within_window(oracle, f) == d
        want = pkg.xxh64(d) & 0xFFFFFFFF
        if checksum:
            assert r["has_checksum"] == 1 and r["checksum"] == want and struct.unpack("<I", f[-4:])[0] == want
        assert r["blocks"] == max(1, -(-len(d) // 131072))
    dec = pkg.FrameDecoder(ctx)
    for d, f in zip(datas, frames):
        assert dec.decode_all(f, len(d)) == d


def batch_decode(pkg, ctx, datas, frames):
    io = np.zeros(len(frames), dtype=pkg.binding.FRAME_IO_DTYPE)
    so = oo = 0
    for i, (f, d) in enumerate(zip(frames, datas)):
        io[i] = (so, len(f), oo, len(d))
        so += len(f)
        oo += len(d)
    out = np.zeros(oo + 16, dtype=np.uint8)
    res = pkg.decode_frames(ctx, np.frombuffer(b"".join(frames), dtype=np.uint8), io, out)
    for i, d in enumerate(datas):
        assert res[i]["status"] == 0 and res[i]["out_size"] == len(d)
        assert out[io[i]["out_off"]:io[i]["out_off"] + len(d)].tobytes() == d


@pytest.mark.parametrize("level", [0, 1])
def test_round_trip_one_batch(pkg, ctx, oracle, inputs, level, monkeypatch):
    names = sorted(inputs)
    datas = [inputs[n] for n in names]
    frames, res = compress_many(pkg, ctx, datas, level)
    check_frames(pkg, ctx, oracle, datas, frames, res)
    for mode in ("cta", "warp"):
        monkeypatch.setenv("B200Z_EXEC_MODE", mode)
        batch_decode(pkg, ctx, datas, frames)
    by = dict(zip(names, zip(frames, res)))
    if level == 1:
        assert by["rle300k"][1]["rle_blocks"] == 3
        assert by["random1m"][1]["raw_blocks"] == 8
        assert len(by["text8m7"][0]) < len(inputs["text8m7"]) // 2


@pytest.mark.parametrize("name", ["size0", "size1", "size5", "size131071", "size131073", "text8m7", "rle300k"])
def test_round_trip_alone_and_device_resident(pkg, ctx, oracle, inputs, name):
    d = inputs[name]
    frames, res = compress_many(pkg, ctx, [d], device=True)
    check_frames(pkg, ctx, oracle, [d], frames, res)
    assert pkg.compress_to_vec(ctx, d) == frames[0]
    plain = pkg.compress_to_vec(ctx, d, checksum=False)
    assert datagen.decompress(plain, len(d)) == d and oracle.decode_frame(plain)[0] == d


def test_deterministic_across_runs_and_batches(pkg, ctx, inputs):
    a = [inputs["text8m7"], inputs["silesia"], inputs["size5"]]
    f1, _ = compress_many(pkg, ctx, a)
    f2, _ = compress_many(pkg, ctx, a)
    assert f1 == f2
    f3, _ = compress_many(pkg, ctx, [inputs["records"], inputs["silesia"], inputs["text128k"], inputs["text8m7"]], device=True)
    assert f3[1] == f1[1] and f3[3] == f1[0]


def test_ratio_floor_on_c2b_shaped_frames(pkg, ctx, oracle):
    plain = datagen.c2_text_plain(64 * 131072).tobytes()
    datas = [plain[i:i + 131072] for i in range(0, len(plain), 131072)]
    frames, res = compress_many(pkg, ctx, datas)
    check_frames(pkg, ctx, oracle, datas[:4], frames[:4], res[:4])
    ratio = len(plain) / sum(len(f) for f in frames)
    zstd1 = len(plain) / sum(len(datagen.compress(d, level=1)) for d in datas)
    print(f"ratio on 64 x 128 KiB gen_text frames: {ratio:.3f} (libzstd level 1: {zstd1:.3f})")
    assert ratio >= 2.2


def test_uncompressed_level_is_header_raw_blocks_checksum(pkg, ctx, inputs):
    for name in ("size0", "size5", "size131073", "text8m7"):
        d = inputs[name]
        n = len(d)
        fcs = struct.pack("<H", n - 256) if 256 <= n <= 65791 else struct.pack("<I", n)
        flag = 1 if len(fcs) == 2 else 2
        want = struct.pack("<IBB", 0xFD2FB528, (flag << 6) | 4, 7 << 3) + fcs
        pieces = [d[i:i + 131072] for i in range(0, n, 131072)] or [b""]
        for k, p in enumerate(pieces):
            want += struct.pack("<I", (1 if k == len(pieces) - 1 else 0) | (len(p) << 3))[:3] + p
        want += struct.pack("<I", pkg.xxh64(d) & 0xFFFFFFFF)
        assert pkg.compress_to_vec(ctx, d, level=pkg.UNCOMPRESSED) == want


def test_rejections_before_any_launch(pkg, ctx):
    L = pkg.lib()
    err = {v: k for k, v in pkg.error_names().items()}
    src = np.zeros(1000, dtype=np.uint8)
    out = np.zeros(4096, dtype=np.uint8)
    bound = pkg.compress_bound(1000)

    def call(rows, level=1, out_arr=out):
        io = np.array(rows, dtype=pkg.binding.COMPRESS_IO_DTYPE)
        res = np.zeros(len(io), dtype=pkg.binding.COMPRESS_RESULT_DTYPE)
        return L.b200z_compress_frames_batch(ctx.h, src.ctypes.data, src.size, 0, io.ctypes.data, len(io), level, 1, out_arr.ctypes.data,
                                             out_arr.size, 0, res.ctypes.data)

    before = ctx.kernel_launches()
    assert call([(0, 1000, 0, bound - 1)]) == err["B200Z_ERR_INVALID_ARGUMENT"]
    assert call([(1, 1000, 0, bound)]) == err["B200Z_ERR_INVALID_ARGUMENT"]
    assert call([(0, 1000, 4096 - bound + 1, bound)]) == err["B200Z_ERR_INVALID_ARGUMENT"]
    assert call([(0, 500, 0, bound), (500, 500, bound - 1, bound)]) == err["B200Z_ERR_INVALID_ARGUMENT"]
    assert call([(0, 1000, 0, bound)], level=9) == err["B200Z_ERR_INVALID_ARGUMENT"]
    for level in (2, 3, 4):
        assert call([(0, 1000, 0, bound)], level=level) == err["B200Z_ERR_REFERENCE_WOULD_PANIC"]
    assert ctx.kernel_launches() == before
    assert call([(0, 500, 0, bound), (500, 500, bound, bound)]) == 0


def test_profile_reports_every_kernel(pkg, ctx, inputs):
    ctx.set_flags(pkg.binding.FLAG_PROFILE)
    try:
        compress_many(pkg, ctx, [inputs["text8m7"]])
        prof = pkg.compress_profile(ctx)
    finally:
        ctx.set_flags(0)
    assert list(prof) == ["k_cmatch", "k_cenc", "k_cxxh64", "k_cassemble"] and all(v >= 0 for v in prof.values())
