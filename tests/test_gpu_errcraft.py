"""Every crafted invalid frame of tests/errcraft.py through every decoding entry, with both execution kernels: the error leaf, stage
and failing block must be the reference's, the bytes before the error must be the reference's, and nothing may be written past a
frame's room.

  batch entry, host and device input (device input is walked by k_walk), device and host output: all cases in one call, each
      between valid frames, with 0xAB guard bytes after every output slot;
  decode_all / decode_all_batch: a valid frame, then the case (then another valid frame unless the case is a frame cut short);
  decode_all_stream: the same bytes in 16 KiB chunks, one block per submission, so a later block's error lands on carried state;
  FrameDecoder: decode_blocks(All) and decode_from_to, then collect, against the oracle doing the same;
  StreamingDecoder: reads of 1000 bytes, against the oracle's StreamingDecoder;
  decode_blocks (the block batch): the cases whose fault lies past the section headers, all in one submission;
  Dictionary.decode_dict: truncated and bad-magic dictionaries, against the oracle's add_dict."""
import numpy as np
import pytest

import errcraft as X
import refwalk

pytestmark = pytest.mark.gpu
GUARD = 0xAB


@pytest.fixture(params=["cta", "warp"])
def exec_mode(request, monkeypatch):
    monkeypatch.setenv("B200Z_EXEC_MODE", request.param)
    return request.param


@pytest.fixture(scope="module")
def crafted():
    return X.cases()


@pytest.fixture(scope="module")
def good():
    return X.good_frames()


def _name(pkg, code):
    return pkg.error_names()[int(code)].replace("B200Z_ERR_", "")


def _oracle_name(oracle, code):
    return oracle.error_names()[code].replace("ZO_ERR_", "")


@pytest.mark.parametrize("device_input,host_output", [(False, False), (True, False), (False, True), (True, True)],
                         ids=["host-input", "device-input", "host-input-host-output", "device-input-host-output"])
def test_batch_between_valid_frames(pkg, ctx, crafted, good, exec_mode, device_input, host_output, monkeypatch):
    """Host input with host output and 64 frames or more takes the pipelined path (1 MiB chunks here: several chunks); device input
    with host output the one-submission path.  Either copies back only what each frame's slot holds."""
    import torch
    monkeypatch.setenv("B200Z_PIPELINE_CHUNK_BYTES", str(1 << 20))
    frames = []                              # (bytes, plaintext or None, case or None)
    for i, c in enumerate(crafted):
        g = good[i % len(good)]
        frames += [(g[0], g[1], None), (c.frame, None, c)]
    frames.append((good[0][0], good[0][1], None))
    io = np.zeros(len(frames), dtype=pkg.binding.FRAME_IO_DTYPE)
    src, oo = bytearray(), 0
    for i, (data, plain, c) in enumerate(frames):
        cap = len(plain) if c is None else c.cap
        io[i] = (len(src), len(data), oo, cap)
        src += data
        oo = (oo + cap + 64 + 127) & ~127
    comp = np.frombuffer(bytes(src), dtype=np.uint8)
    if device_input:
        comp = torch.from_numpy(comp.copy()).cuda()
    assert len(frames) >= 64
    if host_output:
        out = np.full(oo, GUARD, dtype=np.uint8)
        res = pkg.decode_frames(ctx, comp, io, out)
    else:
        d_out = torch.full((oo,), GUARD, dtype=torch.uint8, device="cuda")
        b = pkg.Batch(ctx, comp, io)
        b.run(d_out)
        res = b.finish()
        b.close()
        out = d_out.cpu().numpy()
    for i, (data, plain, c) in enumerate(frames):
        r, o = res[i], int(io[i]["out_off"])
        if c is None:
            assert r["status"] == 0 and r["out_size"] == len(plain) and out[o:o + len(plain)].tobytes() == plain, (i, frames[i - 1][2])
        else:
            assert (_name(pkg, r["status"]), int(r["stage"])) == (c.leaf, c.stage), (c, r)
            if c.stage > X.FRAME_HEADER:
                assert r["error_block"] == c.error_block, (c, r)
        end = o + int(io[i]["out_cap"])
        nxt = int(io[i + 1]["out_off"]) if i + 1 < len(frames) else len(out)
        assert (out[end:nxt] == GUARD).all(), (i, c, "written past out_cap")


def _all_input(c, good):
    g0, g1 = good[0], good[1]
    data = g0[0] + c.frame + (b"" if c.at_end else g1[0])
    return data, g0


def _check_summary(pkg, s, c, g0):
    assert (_name(pkg, s["status"]), s["stage"]) == (c.leaf, c.stage), (c, s)
    assert s["error_frame"] == 1 and s["error_offset"] == len(g0[0]) and s["frames"] == 1, (c, s)
    assert s["written"] == len(g0[1]), (c, s)


def test_decode_all(pkg, ctx, crafted, good, exec_mode):
    import torch
    for c in crafted:
        data, g0 = _all_input(c, good)
        d_out = torch.full((len(g0[1]) + c.cap,), GUARD, dtype=torch.uint8, device="cuda")
        s, _ = pkg.decode_all(ctx, data, d_out)
        _check_summary(pkg, s, c, g0)
        assert d_out[:len(g0[1])].cpu().numpy().tobytes() == g0[1], c


def test_decode_all_batch(pkg, ctx, crafted, good, exec_mode):
    for c in crafted:
        data, g0 = _all_input(c, good)
        out = np.full(len(g0[1]) + c.cap, GUARD, dtype=np.uint8)
        s = pkg.decode_all_batch(ctx, np.frombuffer(data, dtype=np.uint8), out)
        _check_summary(pkg, s, c, g0)
        assert out[:len(g0[1])].tobytes() == g0[1], c


def test_decode_all_stream(pkg, ctx, crafted, good, exec_mode, monkeypatch):
    """16 KiB chunks hold one block each: a later block's fault is decoded in a later submission than its frame's header, from the
    tables, offsets and window the earlier submissions carried over."""
    chunk = 16384
    monkeypatch.setenv("B200Z_PIPELINE_CHUNK_BYTES", str(chunk))
    for c in crafted:
        data, g0 = _all_input(c, good)
        if c.error_block and not c.at_end:
            cuts, _ = pkg.binding.stream_cut(data, chunk)
            at = lambda off: next(k for k, r in enumerate(cuts) if r["start"] <= off < r["end"])
            assert at(len(g0[0]) + c.fault_at) > at(len(g0[0])), c
        drain = bytearray()
        r = pkg.decode_all_stream(ctx, data, drain)
        _check_summary(pkg, r, c, g0)
        assert bytes(drain) == g0[1] + c.prefix_plain and r["delivered"] == len(drain), (c, len(drain))


def _outcome(fn, err_type, name):
    try:
        fn()
    except err_type as e:
        return name(e.code), e.stage
    return None


def test_frame_decoder(pkg, ctx, oracle, crafted, exec_mode):
    for c in crafted:
        for how in ("decode_blocks", "decode_from_to"):
            got = []
            for dec, err_type, name in ((pkg.FrameDecoder(ctx), pkg.B200ZError, lambda k: _name(pkg, k)),
                                        (oracle.FrameDecoder(), oracle.OracleError, lambda k: _oracle_name(oracle, k))):
                if how == "decode_blocks":
                    fn = lambda: dec.decode_blocks(dec.reset(c.frame), pkg.ALL)
                else:
                    fn = lambda: dec.decode_from_to(c.frame, c.cap)
                got.append((_outcome(fn, err_type, name), dec.collect()))
            assert got[0][0] == got[1][0], (c, how, got[0][0], got[1][0])
            # decode_from_to stops without an error where its slice ends inside a block (frame_decoder.rs:479-492)
            if how == "decode_blocks" or not c.at_end:
                assert got[0][0] == (c.leaf, c.stage), (c, how)
            assert got[0][1] == got[1][1], (c, how, len(got[0][1]), len(got[1][1]))


def test_streaming_decoder(pkg, ctx, oracle, crafted, exec_mode):
    for c in crafted:
        got = []
        for mk, err_type, name in ((lambda: pkg.StreamingDecoder(ctx, c.frame), pkg.B200ZError, lambda k: _name(pkg, k)),
                                   (lambda: oracle.StreamingDecoder(c.frame), oracle.OracleError, lambda k: _oracle_name(oracle, k))):
            out = bytearray()

            def run():
                s = mk()
                while True:
                    b = s.read(1000)
                    if not b:
                        return
                    out.extend(b)
            r = _outcome(run, err_type, name)
            got.append((r and r[0], bytes(out)))
        assert got[0] == got[1] and got[0][0] == c.leaf, (c, got[0][0], got[1][0], len(got[0][1]), len(got[1][1]))


def test_block_batch(pkg, ctx, crafted, exec_mode):
    B = pkg.binding
    cs = [c for c in crafted if c.block_level]
    caps = [c.cap for c in cs]
    offs = list(np.cumsum([0] + [cap + 64 for cap in caps[:-1]]))
    comp, blocks, fr = refwalk.walk([c.frame for c in cs], offs, caps, (B.BLOCK_DESC_DTYPE, B.BLOCK_FRAME_DTYPE))
    out = np.full(int(offs[-1]) + caps[-1] + 64, GUARD, dtype=np.uint8)
    st, fo = pkg.decode_blocks(ctx, blocks, fr, comp, out)
    for i, c in enumerate(cs):
        first = int(fr[i]["first_block"])
        for k in range(c.error_block):
            assert st[first + k]["status"] == 0, (c, k)
        s = st[first + c.error_block]
        assert (_name(pkg, s["status"]), int(s["stage"])) == (c.leaf, c.stage), (c, s)
        o = int(offs[i])
        assert out[o:o + len(c.prefix_plain)].tobytes() == c.prefix_plain, c
        assert (out[o + caps[i]:o + caps[i] + 64] == GUARD).all(), (c, "written past out_cap")


def test_dictionaries(pkg, ctx, oracle):
    dicts, good_raw = X.dictionaries()
    pkg.Dictionary.decode_dict(ctx, good_raw)
    for name, raw, leaf in dicts:
        with pytest.raises(pkg.B200ZError) as e:
            pkg.Dictionary.decode_dict(ctx, raw)
        with pytest.raises(oracle.OracleError) as o:
            oracle.FrameDecoder().add_dict(raw)
        assert _name(pkg, e.value.code) == _oracle_name(oracle, o.value.code) == leaf, name
        dec = pkg.FrameDecoder(ctx)
        with pytest.raises(pkg.B200ZError) as e:
            dec.add_dict(raw)
        assert _name(pkg, e.value.code) == leaf, name


def test_frame_decoder_before_init(pkg, ctx, oracle):
    """decode_blocks on a decoder that has not read a frame header: NOT_YET_INITIALIZED, as FrameDecoder::decode_blocks
    (frame_decoder.rs:309-316) reports it."""
    dec = pkg.FrameDecoder(ctx)
    with pytest.raises(pkg.B200ZError) as e:
        dec.decode_blocks(pkg.binding._Reader(b""), pkg.ALL)
    with pytest.raises(oracle.OracleError) as o:
        oracle.FrameDecoder().decode_blocks(oracle._Reader(b""), oracle.ALL)
    assert _name(pkg, e.value.code) == _oracle_name(oracle, o.value.code) == "NOT_YET_INITIALIZED"


def test_frame_decoder_after_an_error(pkg, ctx, oracle, exec_mode):
    """A frame whose failing block leaves a half-built table, then a block that reads it.  The reference reads on when decode_blocks
    is called again and panics (the oracle reports REFERENCE_WOULD_PANIC); the library returns the first error again, as
    include/b200zstd.h documents, and so does a StreamingDecoder read again."""
    for r in X.reentries():
        dec, odec = pkg.FrameDecoder(ctx), oracle.FrameDecoder()
        src, osrc = dec.reset(r.frame), odec.reset(r.frame)
        for want_lib, want_ref in ((r.first, r.first), (r.first, r.second)):
            assert _outcome(lambda: dec.decode_blocks(src, pkg.ALL), pkg.B200ZError, lambda k: _name(pkg, k)) == want_lib, r
            assert _outcome(lambda: odec.decode_blocks(osrc, oracle.ALL), oracle.OracleError, lambda k: _oracle_name(oracle, k)) == want_ref, r
        s = pkg.StreamingDecoder(ctx, r.frame)
        for _ in range(2):
            with pytest.raises(pkg.B200ZError) as e:
                s.read(1000)
            assert _name(pkg, e.value.code) == r.first[0], r
