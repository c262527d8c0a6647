"""The ULTRA level on the GPU against its plain model (tests/cultra.py): every frame is the model's reference_frame byte for byte at
window_log 17, 18, 20, 23 and 27, with and without dictionaries; at window_log 17 it is also GPU OPT's frame.  A mixed submission
(frames below and above 131072 bytes, input ranges out of order and overlapping) gives the same frames in one group and in groups
of a few blocks; the stream compressor writes the batch's blocks; the seekable writers write OPT's archive; the frames round-trip;
launch counts follow the header's formula; levels 6, 8, 9 and 11 are refused before any launch; and the ratio on the ratio input
is the model's."""
import functools
import hashlib
import struct

import numpy as np
import pytest

import cparse
import cultra
import datagen
import streamframe as SF
import test_gpu_cldm as G
from test_gpu_compress_stream import Sink, Source, _chunk
from test_gpu_cparse import compress

pytestmark = pytest.mark.gpu

B = cparse.BLOCK
MIB = 1 << 20
LDM, FAR, STAGES = 17, 14, 4   # long-match kernels, far-stage kernels per group, the four stages (k_copt once per group)

# the model's frame of the ratio input (4 MiB of datagen.gen_text(4 << 20, 0xE90001), window_log 22, checksum): test_cultra_model
# computes it and checks its ratio against OPT's and libzstd level 3's
RATIO_FRAME_LEN = 1161034
RATIO_FRAME_SHA = "d8a842ea7ec957fbc8e9f8ad99c5e436a7ce422d58cfbd8700023b283b50c040"


def ultra(pkg, ctx, datas, **kw):
    return compress(pkg, ctx, datas, level=pkg.ULTRA, **kw)


@functools.lru_cache(None)
def inputs():
    """A 1 MiB frame with repeats 131073, 300,000 and 700,000 bytes back (the last beyond its 2^20 window), 100,000 bytes, and one
    block of the first."""
    big = G.planted(MIB + 3001, 91, [131073, 300000, 700000])
    return [big, G.planted(100000, 92, []), big[:B]]


_models = {}


def model(frames, wl, content=None):
    key = (tuple(map(hash, frames)), wl, content and hash(content))
    if key not in _models:
        _models[key] = cultra.parse(frames, wl, content)
    return _models[key]


@pytest.mark.parametrize("window_log", [17, 18, 20, 23, 27])
def test_frames_are_the_models(pkg, ctx, oracle, window_log):
    plain = inputs()
    blocks = model(plain, window_log)
    before = ctx.kernel_launches()
    frames, _ = ultra(pkg, ctx, plain, window_log=window_log)
    assert ctx.kernel_launches() - before == (STAGES if window_log == 17 else LDM + FAR + STAGES)
    for i, (d, f) in enumerate(zip(plain, frames)):
        assert f == cultra.reference_frame(d, blocks[i], window_log), f"frame {i}"
    if window_log == 17:
        assert frames == compress(pkg, ctx, plain, level=pkg.OPT, window_log=17)[0]
    else:
        assert frames[1:] == compress(pkg, ctx, plain[1:], level=pkg.OPT, window_log=window_log)[0]   # Wf = 131072: OPT's frames
        G.check_decodes(pkg, ctx, oracle, plain, frames, window_log)
    dev, _ = ultra(pkg, ctx, plain[:1], window_log=window_log, checksum=False, device=True)
    assert dev[0] == cultra.reference_frame(plain[0], blocks[0], window_log, checksum=False)


def test_frames_with_dictionaries_are_the_models(pkg, ctx):
    big = inputs()[0]
    content = big[:60000] + bytes(datagen.gen_text(50000, 93))
    datas = [big, big[:200000]]
    blocks = model(datas, 23, content)
    R = pkg.Dictionary.raw_content(ctx, 1, content)
    frames, _ = ultra(pkg, ctx, datas, dict=R, window_log=23)
    for i, d in enumerate(datas):
        assert frames[i] == cultra.reference_frame(d, blocks[i], 23), f"raw content frame {i}"
    fin = pkg.finalize_dict(ctx, content, [big[i:i + 4096] for i in range(0, 400000, 4096)])
    F = pkg.Dictionary.decode_dict(ctx, fin)
    for tables in (False, True):
        frames, _ = ultra(pkg, ctx, datas, dict=F, dict_tables=tables, window_log=23)
        for i, d in enumerate(datas):
            want = cultra.reference_frame(d, blocks[i], 23, dict_id=F.id, dict_tables=fin if tables else None)
            assert frames[i] == want, f"formatted frame {i} tables={tables}"


def mixed(pkg, ctx, big, small, window_log):
    """big and small frames whose input ranges are out of order and overlap: frames [big[300000:], small, big, big[:B + 1]]."""
    src = np.frombuffer(small + big, dtype=np.uint8)
    spans = [(len(small) + 300000, len(big) - 300000), (0, len(small)), (len(small), len(big)), (len(small), B + 1)]
    io = np.zeros(len(spans), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    oo = 0
    for i, (so, n) in enumerate(spans):
        io[i] = (so, n, oo, pkg.compress_bound(n))
        oo += pkg.compress_bound(n)
    out = np.zeros(oo, dtype=np.uint8)
    before = ctx.kernel_launches()
    res = pkg.compress_frames(ctx, src, io, out, pkg.ULTRA, True, window_log=window_log)
    launches = ctx.kernel_launches() - before
    assert (res["status"] == 0).all()
    frames = [out[io[i]["dst_off"]:io[i]["dst_off"] + res[i]["dst_size"]].tobytes() for i in range(len(spans))]
    return [src[so:so + n].tobytes() for so, n in spans], frames, launches


def test_mixed_submission_in_one_group_and_in_several(pkg, ctx, monkeypatch):
    big, small = inputs()[0], inputs()[1]
    _chunk(monkeypatch, None)
    datas, frames, launches = mixed(pkg, ctx, big, small, 23)
    assert launches == LDM + FAR + STAGES
    blocks = model(datas, 23)
    for i, d in enumerate(datas):
        assert frames[i] == cultra.reference_frame(d, blocks[i], 23), f"frame {i}"
    far = [len(d) > B for d in datas for _ in range(-(-len(d) // B))]   # per block: its frame's window is beyond 131072
    for chunk in (B, 3 * B + 5):                     # one group per block; groups of three blocks
        _chunk(monkeypatch, chunk)
        per = chunk // B
        groups = [far[i:i + per] for i in range(0, len(far), per)]
        _, again, launches = mixed(pkg, ctx, big, small, 23)
        assert again == frames
        assert launches == LDM + FAR * sum(map(any, groups)) + len(groups) + STAGES - 1


@pytest.mark.parametrize("chunk", [B, MIB, 12 * MIB])
def test_stream_equals_the_batch_blocks(pkg, ctx, monkeypatch, chunk):
    data = G.planted(3 * MIB + 777, 94, [131073, 600000, 2 * MIB + 3])
    _chunk(monkeypatch, None)
    batch = pkg.compress_to_vec(ctx, data, level=pkg.ULTRA, window_log=23)
    _chunk(monkeypatch, chunk)
    fc = pkg.FrameCompressor(ctx, pkg.ULTRA, window_log=23)
    assert fc.compression_level() == pkg.ULTRA
    src, sink = Source(data, "rand", seed=chunk), Sink()
    fc.set_source(src)
    fc.set_drain(sink)
    r = fc.compress()
    frame = bytes(sink.buf)
    assert r["status"] == 0 and r["dst_size"] == len(frame)
    hdr, blocks, tail = SF.split_frame(frame)
    _, bblocks, btail = SF.split_frame(batch)
    assert hdr == struct.pack("<IBB", 0xFD2FB528, 4, (23 - 10) << 3) and tail == btail
    assert [b[1:] for b in blocks] == [b[1:] for b in bblocks]
    assert datagen.decompress(frame, len(data), window_log_max=27) == data


def test_seekable_archive_is_opts(pkg, ctx):
    plain = inputs()[0]
    for fs in (B, 262144):
        assert pkg.compress_seekable(ctx, plain, frame_size=fs, level=pkg.ULTRA) == pkg.compress_seekable(ctx, plain, frame_size=fs, level=pkg.OPT)


def test_deterministic_across_runs_and_group_sizes(pkg, ctx, monkeypatch):
    plain = inputs()
    _chunk(monkeypatch, None)
    a, _ = ultra(pkg, ctx, plain, window_log=27)
    b, _ = ultra(pkg, ctx, plain, window_log=27)
    _chunk(monkeypatch, 2 * B)
    c, _ = ultra(pkg, ctx, plain[::-1], window_log=27)
    assert a == b == c[::-1]


def test_levels_6_8_9_and_11_are_refused_before_any_launch(pkg, ctx):
    L = pkg.lib()
    err = {v: k for k, v in pkg.error_names().items()}
    src = np.zeros(1000, dtype=np.uint8)
    out = np.zeros(4096, dtype=np.uint8)
    io = np.array([(0, 1000, 0, pkg.compress_bound(1000))], dtype=pkg.binding.COMPRESS_IO_DTYPE)
    res = np.zeros(1, dtype=pkg.binding.COMPRESS_RESULT_DTYPE)
    before = ctx.kernel_launches()
    for level in (6, 8, 9, 11):
        assert L.b200z_compress_frames_batch(ctx.h, src.ctypes.data, src.size, 0, io.ctypes.data, 1, level, 1, out.ctypes.data, out.size, 0,
                                             res.ctypes.data) == err["B200Z_ERR_INVALID_ARGUMENT"]
        with pytest.raises(pkg.B200ZError):
            pkg.FrameCompressor(ctx, level)
    fc = pkg.FrameCompressor(ctx, pkg.ULTRA)
    with pytest.raises(pkg.B200ZError):
        fc.set_compression_level(11)
    assert fc.compression_level() == pkg.ULTRA
    assert ctx.kernel_launches() == before


def test_ratio_is_the_models(pkg, ctx):
    data = bytes(datagen.gen_text(4 << 20, 0xE90001))
    frame = pkg.compress_to_vec(ctx, data, level=pkg.ULTRA, window_log=22)
    opt = pkg.compress_to_vec(ctx, data, level=pkg.OPT, window_log=22)
    print(f"ULTRA {len(data) / len(frame):.4f}, OPT {len(data) / len(opt):.4f} at window_log 22")
    assert len(frame) == RATIO_FRAME_LEN and hashlib.sha256(frame).hexdigest() == RATIO_FRAME_SHA
    assert datagen.decompress(frame, len(data), window_log_max=27) == data
