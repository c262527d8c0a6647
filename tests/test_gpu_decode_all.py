"""decode_all on the batch path (b200z_decode_all_prepare / b200z_batch_run / b200z_decode_all_finish): buffers of concatenated
frames decoded in one submission, checked against the oracle's FrameDecoder.decode_all (output bytes, error leaf and stage) and
against the tier-2 FrameDecoder.decode_all."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from conftest import read_golden
from test_decode_all_chain import concat_with_skippables, corpus_frames, raw_frame, skippable

pytestmark = pytest.mark.gpu

IO_MODES = [(False, False), (True, True), (False, True), (True, False)]   # (device input, device output)


@pytest.fixture(params=["cta", "warp"])
def exec_mode(request, monkeypatch):
    """Every test runs with the multi-block frames on k_exec_cta and with everything on k_exec."""
    monkeypatch.setenv("B200Z_EXEC_MODE", request.param)
    return request.param


def oracle_all(oracle, data, cap, dict_raw=None):
    d = oracle.FrameDecoder()
    if dict_raw is not None:
        d.add_dict(dict_raw)
    try:
        return d.decode_all(data, cap), None
    except oracle.OracleError as e:
        return None, (oracle.error_names()[e.code].replace("ZO_", ""), e.stage)


def gpu_all(pkg, ctx, data, cap, dev_in=True, dev_out=True, **kw):
    import torch
    a = np.frombuffer(bytes(data), dtype=np.uint8).copy()
    inp = torch.from_numpy(a).cuda() if dev_in else a
    if dev_out:
        buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
        summary, res = pkg.decode_all(ctx, inp, buf[:cap], **kw)
        out = buf[:summary["written"]].cpu().numpy().tobytes()
    else:
        buf = np.zeros(max(cap, 1), dtype=np.uint8)
        summary, res = pkg.decode_all(ctx, inp, buf[:cap], **kw)
        out = buf[:summary["written"]].tobytes()
    return summary, res, out


def check_against_oracle(pkg, ctx, oracle, data, cap, dev_in=True, dev_out=True, dict_raw=None, **kw):
    exp, exp_err = oracle_all(oracle, data, cap, dict_raw)
    summary, res, out = gpu_all(pkg, ctx, data, cap, dev_in, dev_out, **kw)
    if exp_err is None:
        assert summary["status"] == 0, (summary, len(data), cap)
        assert out == exp
    else:
        got = (pkg.error_names()[summary["status"]].replace("B200Z_", ""), summary["stage"])
        assert got == exp_err, (got, exp_err, summary, len(data), cap)
    return summary, res, out, exp_err


@pytest.mark.parametrize("dev_in,dev_out", IO_MODES)
def test_corpus_concatenation(pkg, ctx, oracle, manifest, exec_mode, dev_in, dev_out):
    frames = corpus_frames(manifest)
    buf, _starts = concat_with_skippables(frames)
    plains = [oracle.decode_frame(f)[0] for f in frames]
    total = sum(len(p) for p in plains)
    summary, res, out, _ = check_against_oracle(pkg, ctx, oracle, buf, total, dev_in, dev_out)
    assert out == b"".join(plains)
    assert summary["frames"] == 101 and summary["skippable_frames"] == 101 and summary["written"] == total
    assert summary["error_offset"] == len(buf) and summary["error_frame"] == -1
    for i, f in enumerate(frames):
        _, d = oracle.decode_frame(f)
        assert res[i]["status"] == 0 and res[i]["out_size"] == len(plains[i]) and res[i]["bytes_read"] == d.bytes_read_from_source()
        assert res[i]["content_size"] == d.content_size()
    if not dev_in and not dev_out:
        assert pkg.FrameDecoder(ctx).decode_all(buf, total) == out


def test_truncations_and_garbage(pkg, ctx, oracle, manifest, exec_mode):
    buf, starts = concat_with_skippables(corpus_frames(manifest)[:12])
    cap = 1 << 22
    cuts = sorted({s + d for s in starts + [len(buf)] for d in (-4, -1, 0, 1, 5) if 0 <= s + d <= len(buf)})
    for i, cut in enumerate(cuts):
        check_against_oracle(pkg, ctx, oracle, buf[:cut], cap, dev_in=i % 2 == 0, dev_out=i % 3 != 0)
    for tail in (b"\x00", b"\x28\xb5", b"\x28\xb5\x2f", b"no frame here", b"\x28\xb5\x2f\xfd", b"\x50\x2a\x4d\x18\x00\x00",
                 b"\x50\x2a\x4d\x18\x10\x00\x00\x00abc"):
        s, _, _, err = check_against_oracle(pkg, ctx, oracle, buf + tail, cap)
        assert err is not None and s["error_offset"] == len(buf)


def test_fuzz_artifacts_appended(pkg, ctx, oracle, manifest, exec_mode):
    head = b"".join(corpus_frames(manifest)[:3])
    for sub, files in manifest["fuzz"].items():
        for i, f in enumerate(files):
            check_against_oracle(pkg, ctx, oracle, head + read_golden("fuzz", sub, f), 1 << 22, dev_in=i % 2 == 0)


def _blocks(frame):
    """(content offset, type, content size, last) of every block of a valid frame."""
    import refwalk
    pos = refwalk.frame_header(frame)[0]
    out = []
    while True:
        h = int.from_bytes(frame[pos:pos + 3], "little")
        t, size = (h >> 1) & 3, h >> 3
        c = 1 if t == 1 else size
        out.append((pos + 3, t, c, h & 1))
        pos += 3 + c
        if h & 1:
            return out


def test_output_cap_sweep(pkg, ctx, oracle, exec_mode):
    import datagen as G
    small = [G.compress(G.gen_text(5000 + 3000 * i, 900 + i).tobytes()) for i in range(3)]
    big_plain = G.gen_text(700000, 911).tobytes()
    big = G.compress(big_plain, window_log=17)
    assert len(_blocks(big)) >= 5
    frames = [small[0], big, small[1], small[2]]
    buf = b"".join(frames)
    sizes = [len(oracle.decode_frame(f)[0]) for f in frames]
    bounds = np.cumsum([0] + sizes).tolist()
    total = bounds[-1]
    caps = {total - 1, total, total + 1}
    for b in bounds[1:-1]:
        caps |= {b - 1, b, b + 1}
    caps |= {bounds[1] + k * 100000 for k in range(1, 7)}
    for i, cap in enumerate(sorted(c for c in caps if c >= 0)):
        check_against_oracle(pkg, ctx, oracle, buf, cap, dev_in=i % 2 == 0, dev_out=i % 3 != 0)
    # a later block of the multi-block frame is broken: TargetTooSmall or the block error, as the UptoBytes / window loop decides
    blocks = _blocks(big)
    reserved = bytearray(big)
    reserved[blocks[4][0] - 3] |= 0x06
    flipped = bytearray(big)
    o = blocks[3][0]
    flipped[o] ^= 0xFF
    for broken in (bytes(reserved), bytes(flipped)):
        b2 = small[0] + broken + small[1]
        for cap in sorted({bounds[1] + k * 65536 for k in range(0, 11)} | {total}):
            check_against_oracle(pkg, ctx, oracle, b2, cap)
        assert pkg.FrameDecoder(ctx).decode_all(small[0], sizes[0]) == oracle.decode_frame(small[0])[0]


def _compress_no_content_size(data):
    import datagen as G
    z = G.zstd()
    a = np.frombuffer(data, dtype=np.uint8)
    cap = z.ZSTD_compressBound(a.nbytes)
    dst = np.empty(cap, dtype=np.uint8)
    cctx = z.ZSTD_createCCtx()
    try:
        z.ZSTD_CCtx_setParameter(cctx, 100, 3)      # ZSTD_c_compressionLevel
        z.ZSTD_CCtx_setParameter(cctx, 200, 0)      # ZSTD_c_contentSizeFlag
        z.ZSTD_CCtx_setParameter(cctx, 201, 1)      # ZSTD_c_checksumFlag
        n = z.ZSTD_compress2(cctx, dst.ctypes.data, cap, a.ctypes.data, a.nbytes)
    finally:
        z.ZSTD_freeCCtx(cctx)
    assert not z.ZSTD_isError(n)
    return dst[:n].tobytes()


def _with_content_size(frame, value):
    """A frame without Frame_Content_Size (not single-segment, no dictionary id) given a 4-byte content-size field holding `value`."""
    assert frame[4] >> 5 == 0 and frame[4] & 3 == 0
    return frame[:4] + bytes([frame[4] | 0x80, frame[5]]) + int(value).to_bytes(4, "little") + frame[6:]


def test_content_size_is_not_used_for_placement(pkg, ctx, oracle, exec_mode):
    import datagen as G
    plains = [G.gen_text(40000 + 20000 * i, 930 + i).tobytes() for i in range(4)]
    no_fcs = [_compress_no_content_size(p) for p in plains]
    assert all(f[4] >> 6 == 0 for f in no_fcs)
    buf = b"".join(no_fcs)
    s, _, out, _ = check_against_oracle(pkg, ctx, oracle, buf, sum(map(len, plains)) + 100)
    assert out == b"".join(plains)
    # a Frame_Content_Size smaller / larger than the content: placement still follows the decoded sizes
    lied = [_with_content_size(f, len(p) // 2 if i % 2 else len(p) * 3) for i, (f, p) in enumerate(zip(no_fcs, plains))]
    for dev_in in (False, True):
        s, res, out, _ = check_against_oracle(pkg, ctx, oracle, b"".join(lied), sum(map(len, plains)), dev_in=dev_in)
        assert out == b"".join(plains) and list(res["out_size"]) == [len(p) for p in plains]
        assert list(res["content_size"]) == [len(p) // 2 if i % 2 else len(p) * 3 for i, p in enumerate(plains)]


def test_false_candidates_in_uncompressed_frame(pkg, ctx, oracle, manifest, exec_mode):
    frames = corpus_frames(manifest)[:8]
    inner = b"".join(frames) + skippable(7)
    wrapped = pkg.compress_to_vec(ctx, inner, level=pkg.UNCOMPRESSED)
    assert inner.count(b"\x28\xb5\x2f\xfd") >= 8
    buf = frames[0] + wrapped + frames[1] + raw_frame(inner) + frames[2]
    plains = [oracle.decode_frame(f)[0] for f in frames[:3]]
    want = plains[0] + inner + plains[1] + inner + plains[2]
    for dev_in in (False, True):
        s, res, out, _ = check_against_oracle(pkg, ctx, oracle, buf, len(want), dev_in=dev_in)
        assert out == want and s["frames"] == 5


def test_dictionaries(pkg, ctx, oracle, manifest, exec_mode):
    dic = read_golden("dict_tests", "dictionary")
    names = sorted(manifest["dict"])[:60]
    frames = [read_golden("dict_tests", "files", n) for n in names]
    buf = b"".join(f + (skippable(3) if i % 5 == 0 else b"") for i, f in enumerate(frames))
    D = pkg.Dictionary.decode_dict(ctx, dic)
    total = sum(manifest["dict"][n]["size"] for n in names)
    s, res, out, _ = check_against_oracle(pkg, ctx, oracle, buf, total, dict_raw=dic, dicts=[D])
    assert s["frames"] == len(frames) and hashlib.sha256(out).hexdigest() == hashlib.sha256(
        b"".join(oracle.decode_frame(f, dict_raw=dic)[0] for f in frames)).hexdigest()
    # no dictionary: DictNotProvided at the first frame; a frame without dictionary id first, then a dictionary frame
    s, _, _, _ = check_against_oracle(pkg, ctx, oracle, buf, total)
    assert pkg.error_names()[s["status"]] == "B200Z_ERR_DICT_NOT_PROVIDED" and s["error_frame"] == 0 and s["error_offset"] == 0
    head = b"".join(corpus_frames(manifest)[:2])
    s, _, _, _ = check_against_oracle(pkg, ctx, oracle, head + buf, 1 << 22)
    assert s["error_frame"] == 2 and s["error_offset"] == len(head)


def test_forced_raw_content_dictionary(pkg, ctx, exec_mode):
    """C5-shaped frames (raw-content dictionary, no dictionary id) through the forced_dict extension."""
    import datagen as G
    fs = G.config_c5(nframes=300, cache=False)
    D = pkg.Dictionary.raw_content(ctx, 1, fs.raw_dict)
    s, res, out = gpu_all(pkg, ctx, fs.comp.tobytes(), fs.D, forced_dict=D)
    assert s["status"] == 0 and s["frames"] == 300 and out == fs.plain.tobytes()


def test_window_fixture_twice(pkg, ctx, oracle, exec_mode):
    big = read_golden("test_fixtures", "window_256mib.zst")
    buf = big + big
    fox_len = len(pkg.FrameDecoder(ctx).decode_all(read_golden("test_fixtures", "window_128mib.zst"), 1 << 20))
    s, _, _, _ = check_against_oracle(pkg, ctx, oracle, buf, 2 * fox_len + 100)
    assert pkg.error_names()[s["status"]] == "B200Z_ERR_WINDOW_SIZE_TOO_BIG" and s["error_frame"] == 0
    s, res, out = gpu_all(pkg, ctx, buf, 2 * fox_len + 100, max_window_size=1 << 29)
    assert s["status"] == 0 and s["frames"] == 2 and out[:fox_len] == out[fox_len:]


def test_empty_and_skippable_only(pkg, ctx, oracle, exec_mode):
    for buf in (b"", skippable(0), skippable(0) + skippable(300, 15) + skippable(1, 3)):
        s, res, out, _ = check_against_oracle(pkg, ctx, oracle, buf, 64)
        assert s["status"] == 0 and s["written"] == 0 and s["frames"] == 0 and len(res) == 0


@pytest.mark.parametrize("checksum_flag", [False, True])
def test_round_trip_compressed_frames(pkg, ctx, exec_mode, checksum_flag):
    import datagen as G
    plains = [G.gen_text(1000 + 37000 * i, 950 + i).tobytes() for i in range(12)]
    src = b"".join(plains)
    io = np.zeros(len(plains), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    so = do = 0
    for i, p in enumerate(plains):
        cap = pkg.compress_bound(len(p))
        io[i] = (so, len(p), do, cap)
        so += len(p); do += cap
    out = np.zeros(do, dtype=np.uint8)
    r = pkg.compress_frames(ctx, src, io, out)
    packed = b"".join(out[io[i]["dst_off"]:io[i]["dst_off"] + r[i]["dst_size"]].tobytes() for i in range(len(plains)))
    c2 = pkg.Context(0)
    if checksum_flag:
        c2.set_flags(pkg.binding.FLAG_CHECKSUM)
    s, res, got = gpu_all(pkg, c2, packed, len(src))
    assert s["status"] == 0 and got == src
    if checksum_flag:
        assert (res["has_calculated_checksum"] == 1).all() and (res["calculated_checksum"] == res["checksum_from_data"]).all()
    c2.close()


@pytest.mark.parametrize("config", ["c2b", "c4", "c5"])
def test_small_configs_and_launch_counts(pkg, config, monkeypatch):
    import torch
    import datagen as G
    fs = {"c2b": lambda: G.config_c2b(total_bytes=64 << 20, cache=False), "c4": lambda: G.config_c4(nframes=16, cache=False),
          "c5": lambda: G.config_c5(nframes=2000, cache=False)}[config]()
    for mode in ("warp", "cta"):
        monkeypatch.setenv("B200Z_EXEC_MODE", mode)
        c2 = pkg.Context(0)
        D = pkg.Dictionary.raw_content(c2, 1, fs.raw_dict) if fs.raw_dict is not None else None
        d_in = torch.from_numpy(fs.comp.copy()).cuda()
        out = torch.zeros(fs.D + 16, dtype=torch.uint8, device="cuda")
        ab = pkg.AllBatch(c2, d_in, forced_dict=D)
        assert ab.info()["frames"] == fs.nframes
        ab.run(out[:fs.D])
        s, res = ab.finish()
        assert s["status"] == 0 and s["written"] == fs.D and out[:fs.D].cpu().numpy().tobytes() == fs.plain.tobytes()
        # the known-offset batch on the same frames launches the same kernels, k_place aside
        io = np.zeros(fs.nframes, dtype=pkg.binding.FRAME_IO_DTYPE)
        io["src_off"], io["src_size"], io["out_off"], io["out_cap"] = fs.src_off, fs.src_size, fs.out_off, fs.out_size
        kb = pkg.Batch(c2, d_in, io, forced_dict=D)
        kb.run(out[:fs.D])
        n_cta = kb.debug_sched()["cta_frames"]
        expect = 4 + (1 if n_cta < fs.nframes else 0) + (2 if n_cta else 0)
        assert kb.info()["launches_per_run"] == expect
        assert ab.info()["launches_per_run"] == expect + 1
        ab.close(); kb.close()
        c2.close()
