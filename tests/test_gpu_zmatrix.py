"""The libzstd matrix (tests/zmatrix.py) on the GPU, with the multi-block frames on k_exec_cta, everything on k_exec, and the
shipped routing: every frame in one submission and the large ones alone, with checksums, canaries after every slot and each
Compressed block's literals and sequences against the oracle's trace; device input at every address residue through k_walk and
k_find_frames; decode_all and decode_all_stream over the multi-frame buffers; the tier-2 FrameDecoder and StreamingDecoder; and
the dictionary frames by ID and forced."""
import random
import time

import numpy as np
import pytest

import intermediates
import zmatrix as Z
from test_gpu_decode_all_stream import SUMMARY, Drain, stream

pytestmark = pytest.mark.gpu

CANARY = 16


@pytest.fixture(params=["cta", "warp", "auto"])
def exec_mode(request, monkeypatch):
    """cta: the frames without a dictionary on k_exec_cta; warp: everything on k_exec; auto: the shipped routing."""
    if request.param == "auto":
        monkeypatch.delenv("B200Z_EXEC_MODE", raising=False)
    else:
        monkeypatch.setenv("B200Z_EXEC_MODE", request.param)
    return request.param


@pytest.fixture(scope="module")
def matrix(oracle):
    t = time.time()
    fs = Z.frames()
    _, exact = Z.census(oracle, fs)
    yield fs, exact
    print(f"\nzmatrix: {len(fs)} frames, {sum(len(f.plain) for f in fs) / Z.MiB:.1f} MiB; module wall time {time.time() - t:.1f} s")


@pytest.fixture(scope="module")
def dicts(pkg, ctx):
    D = pkg.Dictionary.decode_dict(ctx, Z.trained_dict())
    assert D.id == Z.trained_dict_id()
    return D, pkg.Dictionary.raw_content(ctx, 1, Z.raw_dict_content())


@pytest.fixture
def checksum_flag(pkg, ctx):
    old = ctx.L.b200z_ctx_flags(ctx.h)
    ctx.set_flags(old | pkg.binding.FLAG_CHECKSUM)
    yield
    ctx.set_flags(old)


def submissions(fs, dicts):
    """The frames split by how their dictionary reaches the decoder: by ID (and no dictionary), forced formatted, forced raw."""
    D, R = dicts
    return [([f for f in fs if f.dict is None or f.dict_id], dict(dicts=[D]), list(D.offset_hist)),
            ([f for f in fs if f.dict == "formatted" and not f.dict_id], dict(forced_dict=D), list(D.offset_hist)),
            ([f for f in fs if f.dict == "raw"], dict(forced_dict=R), [1, 4, 8])]


def run_batch(pkg, ctx, fs, exec_mode, **kw):
    """One submission of `fs`, each slot followed by CANARY bytes; checks status, sizes, bytes read, checksums, canaries and
    (cta) that k_exec_cta took every frame without a dictionary and handed none back to k_exec.  Returns (the Batch, the
    number of checksums compared)."""
    import torch
    io = np.zeros(len(fs), dtype=pkg.binding.FRAME_IO_DTYPE)
    so = oo = nck = 0
    for i, f in enumerate(fs):
        io[i] = (so, len(f.data), oo, len(f.plain))
        so += len(f.data); oo += len(f.plain) + CANARY
    d_out = torch.full((oo,), 0xAB, dtype=torch.uint8, device="cuda")
    b = pkg.Batch(ctx, np.frombuffer(b"".join(f.data for f in fs), dtype=np.uint8), io, max_window_size=Z.RAISED_MAX_WINDOW, **kw)
    b.run(d_out)
    res = b.finish()
    out = d_out.cpu().numpy()
    for i, f in enumerate(fs):
        r, o = res[i], int(io[i]["out_off"])
        assert r["status"] == 0, (f.id, r)
        assert r["out_size"] == len(f.plain) and r["bytes_read"] == len(f.data), (f.id, r)
        assert out[o:o + len(f.plain)].tobytes() == f.plain, f.id
        assert (out[o + len(f.plain):o + len(f.plain) + CANARY] == 0xAB).all(), f.id
        assert r["has_checksum"] == f.checksum, (f.id, r)
        if f.checksum:
            assert r["has_calculated_checksum"] and r["calculated_checksum"] == r["checksum_from_data"], (f.id, r)
            assert r["checksum_from_data"] == pkg.xxh64(f.plain) & 0xFFFFFFFF, f.id
            nck += 1
    if exec_mode == "cta":
        s = b.debug_sched()
        assert s["cta_frames"] == sum(1 for f in fs if f.dict is None), (s, len(fs))
        assert s["handed_back_frames"] == 0 and s["reasons"] == 0, (s, [f.id for f in fs][:3])
    return b, nck


def test_batch_and_intermediates(pkg, ctx, oracle, matrix, dicts, exec_mode, checksum_flag):
    fs, exact = matrix
    nlit = nseq = nexact = nck = 0
    for group, kw, hist in submissions(fs, dicts):
        b, n = run_batch(pkg, ctx, group, exec_mode, **kw)
        nck += n
        blk = 0
        for f in group:
            _, _, blocks, lits, seqs = Z.trace(oracle, f)
            blk, nl, ns = intermediates.check_intermediates(b, blk, blocks, lits, seqs, f.id, hist=hist if f.dict else (1, 4, 8),
                                                exact=exact[f.id], flags_exact=exec_mode == "warp")
            nlit += nl; nseq += ns; nexact += sum(exact[f.id])
        assert blk == b.info()["blocks"]
        b.close()
    assert nlit > 2000 and nseq > 5_000_000 and nexact >= 1 and nck == sum(f.checksum for f in fs)


def test_large_frames_alone(pkg, ctx, matrix, dicts, exec_mode, checksum_flag):
    fs, _ = matrix
    n = nck = 0
    for group, kw, _ in submissions(fs, dicts):
        for f in group:
            if len(f.plain) >= Z.MiB:
                b, k = run_batch(pkg, ctx, [f], exec_mode, **kw)
                b.close()
                n += 1; nck += k
    assert n >= 30 and nck == n - 1   # all but nochecksum-records


def test_window_limit(pkg, ctx, matrix):
    f = Z.by_id(matrix[0])["wlog28-stream-256MiB-window"]
    io = np.zeros(1, dtype=pkg.binding.FRAME_IO_DTYPE)
    io[0] = (0, len(f.data), 0, len(f.plain))
    out = np.zeros(len(f.plain) + 16, dtype=np.uint8)
    res = pkg.decode_frames(ctx, np.frombuffer(f.data, dtype=np.uint8), io, out)
    assert pkg.error_names()[int(res[0]["status"])] == "B200Z_ERR_WINDOW_SIZE_TOO_BIG"
    res = pkg.decode_frames(ctx, np.frombuffer(f.data, dtype=np.uint8), io, out, max_window_size=Z.RAISED_MAX_WINDOW)
    assert res[0]["status"] == 0 and out[:len(f.plain)].tobytes() == f.plain


def test_device_input_at_every_residue(pkg, ctx, matrix, exec_mode):
    """Device input as big[r : r + n] for r = 0..15: k_walk (decode_frames) and k_find_frames (decode_all) on buffers whose head
    and tail are not 16-byte aligned."""
    import torch
    bufs = Z.multi_frame_buffers(matrix[0])
    by = Z.by_id(matrix[0])
    cat, cat_plain, ids = bufs["concat"]
    io = np.zeros(len(ids), dtype=pkg.binding.FRAME_IO_DTYPE)
    so = oo = 0
    for i, fid in enumerate(ids):
        io[i] = (so, len(by[fid].data), oo, len(by[fid].plain))
        so += len(by[fid].data); oo += len(by[fid].plain)
    host_res = pkg.decode_frames(ctx, np.frombuffer(cat, dtype=np.uint8), io, np.zeros(oo + 16, dtype=np.uint8))
    pz, pz_plain, pz_ids = bufs["pzstd"]
    for r in range(16):
        big = torch.zeros(len(cat) + 32, dtype=torch.uint8, device="cuda")
        big[r:r + len(cat)] = torch.from_numpy(np.frombuffer(cat, dtype=np.uint8).copy())
        d_out = torch.zeros(oo + 16, dtype=torch.uint8, device="cuda")
        res = pkg.decode_frames(ctx, big[r:r + len(cat)], io, d_out)
        for k in res.dtype.names:
            assert np.array_equal(res[k], host_res[k]), (r, k)
        assert d_out[:oo].cpu().numpy().tobytes() == cat_plain, r
        big = torch.zeros(len(pz) + 32, dtype=torch.uint8, device="cuda")
        big[r:r + len(pz)] = torch.from_numpy(np.frombuffer(pz, dtype=np.uint8).copy())
        d_out = torch.zeros(len(pz_plain) + 16, dtype=torch.uint8, device="cuda")
        s, _ = pkg.decode_all(ctx, big[r:r + len(pz)], d_out[:len(pz_plain)])
        assert s["status"] == 0 and s["written"] == len(pz_plain) and s["frames"] == len(pz_ids), (r, s)
        assert s["skippable_frames"] == len(pz_ids) and s["error_offset"] == len(pz), (r, s)
        assert d_out[:len(pz_plain)].cpu().numpy().tobytes() == pz_plain, r


def test_decode_all_and_stream(pkg, ctx, oracle, matrix, exec_mode, monkeypatch):
    for name, (buf, plain, ids) in Z.multi_frame_buffers(matrix[0]).items():
        assert oracle.FrameDecoder().decode_all(buf, len(plain)) == plain, name
        out = np.zeros(len(plain) + 16, dtype=np.uint8)
        s, res = pkg.decode_all(ctx, buf, out[:len(plain)])
        assert out[:len(plain)].tobytes() == plain, name
        want = {"written": len(plain), "frames": len(ids), "skippable_frames": len(ids) if name == "pzstd" else 0,
                "error_offset": len(buf), "status": 0, "stage": s["stage"], "error_frame": -1}
        assert {k: s[k] for k in SUMMARY} == want, (name, s)
        assert (res["status"] == 0).all()
        for chunk in (Z.MiB, None):
            if chunk is None:   # the library's default chunk size
                monkeypatch.delenv("B200Z_PIPELINE_CHUNK_BYTES", raising=False)
                d = Drain()
                r = pkg.decode_all_stream(ctx, buf, d)
                got = bytes(d.out)
            else:
                r, got = stream(pkg, ctx, monkeypatch, buf, chunk)
            assert {k: r[k] for k in SUMMARY} == {k: s[k] for k in SUMMARY}, (name, chunk, r)
            assert got == plain, (name, chunk)
            if chunk == Z.MiB:
                assert r["submissions"] > 1, (name, r)


def test_frame_decoder_every_frame(pkg, ctx, matrix, exec_mode):
    for f in matrix[0]:
        d = pkg.FrameDecoder(ctx)
        r = Z.setup_decoder(d, f)
        assert d.decode_blocks(r, pkg.ALL) is True, f.id
        assert d.collect() == f.plain, f.id
        assert d.bytes_read_from_source() == len(f.data), f.id
        if d.get_checksum_from_data() is not None:
            assert d.get_calculated_checksum() == d.get_checksum_from_data(), f.id


STREAMED = ["wlog10-text-1KiB-blocks", "flushed-text-small-blocks", "tcbs1340-text-treeless", "wlog27-ldm-far-offsets",
            "cdict-level3/0", "cdict-level19/5"]


def test_streaming_decoder_lockstep(pkg, ctx, oracle, matrix, exec_mode):
    by = Z.by_id(matrix[0])
    for fid in STREAMED:
        f = by[fid]
        ga, ob = pkg.FrameDecoder(ctx), oracle.FrameDecoder()
        for d in (ga, ob):
            if f.dict == "formatted":
                d.add_dict(Z.trained_dict())
        a, b = pkg.StreamingDecoder(ctx, f.data, decoder=ga), oracle.StreamingDecoder(f.data, decoder=ob)
        rng = random.Random(fid)
        got = bytearray()
        while True:
            n = rng.choice([1, 7, 1000, 4096, 65536, 200_000, 1 << 20])
            x, y = a.read(n), b.read(n)
            assert x == y, (fid, len(got), n)
            if not y:
                break
            got += y
        assert bytes(got) == f.plain, fid


def test_dictionaries(pkg, ctx, matrix, dicts):
    """By ID with Dictionary.decode_dict; forced where the frame has no ID: the formatted dictionary for the CDict frames written
    without their ID, raw content (under any ID) for the ZSTD_compress_usingDict frames.  Without the dictionary an ID-named frame
    fails with DictNotProvided."""
    D, R = dicts
    fs = matrix[0]
    ided = [f for f in fs if f.dict == "formatted" and f.dict_id]
    noid = [f for f in fs if f.dict == "formatted" and not f.dict_id]
    raw = [f for f in fs if f.dict == "raw"]
    R2 = pkg.Dictionary.raw_content(ctx, 7, Z.raw_dict_content())
    for group, kw in ((ided, dict(dicts=[D])), (noid, dict(forced_dict=D)), (raw, dict(forced_dict=R)), (raw, dict(forced_dict=R2))):
        io = np.zeros(len(group), dtype=pkg.binding.FRAME_IO_DTYPE)
        so = oo = 0
        for i, f in enumerate(group):
            io[i] = (so, len(f.data), oo, len(f.plain))
            so += len(f.data); oo += len(f.plain)
        out = np.zeros(oo + 16, dtype=np.uint8)
        res = pkg.decode_frames(ctx, np.frombuffer(b"".join(f.data for f in group), dtype=np.uint8), io, out, **kw)
        assert (res["status"] == 0).all(), res[res["status"] != 0][:3]
        assert out[:oo].tobytes() == b"".join(f.plain for f in group)
        if group is ided:
            assert (res["has_dict_id"] == 1).all() and (res["dict_id"] == D.id).all()
    # without the dictionary the ID-named frames fail with DictNotProvided
    f = ided[0]
    io = np.zeros(1, dtype=pkg.binding.FRAME_IO_DTYPE); io[0] = (0, len(f.data), 0, len(f.plain))
    res = pkg.decode_frames(ctx, np.frombuffer(f.data, dtype=np.uint8), io, np.zeros(len(f.plain) + 16, dtype=np.uint8))
    assert pkg.error_names()[int(res[0]["status"])] == "B200Z_ERR_DICT_NOT_PROVIDED"
