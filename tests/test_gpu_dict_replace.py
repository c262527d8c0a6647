"""Ownership of the library's resources, seen from outside: a dictionary replaced in a frame decoder while a frame is being
decoded stays with that frame until it ends (the reference copies it into the frame's scratch when the frame starts), and a
stream compressor whose chunks do not fit in device memory fails cleanly and leaves the context usable."""
import pytest

import datagen
import dictcraft as D
from test_gpu_compress_stream import Sink, Source, _err, check_fastest, run

pytestmark = pytest.mark.gpu


def _replacement(d):
    """A dictionary of d's ID and kind (and a formatted one's repeat offsets) with other content of the same length."""
    return D.Dict(d.name + "-replaced", d.id, bytes(b ^ 0x5A for b in d.content), d.reps if d.formatted else None)


def _add(dec, d):
    if d.formatted:
        dec.add_dict(d.raw)
    else:
        dec.add_raw_content_dict(d.id, d.content)


def _decode(mod, dec, frame, replace=None):
    """reset, decode_blocks(UptoBlocks, 1), add `replace`, decode_blocks(All), collect; the same calls on the GPU decoder and the
    oracle's (`mod` is the package or the oracle module)."""
    r = dec.reset(frame)
    dec.decode_blocks(r, mod.UPTO_BLOCKS, 1)
    if replace is not None:
        _add(dec, replace)
    dec.decode_blocks(r, mod.ALL)
    return dec.collect()


def test_dictionary_replaced_mid_frame(pkg, ctx, oracle):
    cs = [c for c in D.cases() if c.valid and c.dict is not None and c.forced is None and len(c.blocks) >= 2]
    assert cs
    differs = 0
    for c in cs:
        g = pkg.FrameDecoder(ctx)
        for d in D.DICTS:
            _add(g, d)
        o = D.oracle_decoder(oracle)
        new = _replacement(c.dict)
        got = _decode(pkg, g, c.frame, new)
        assert got == c.expected, c
        assert _decode(oracle, o, c.frame, new) == got, c
        # the next frame starts from the replacement
        again = _decode(pkg, g, c.frame)
        assert again == _decode(oracle, o, c.frame), c
        differs += again != c.expected
    assert differs, "no selected case depends on its dictionary's content"


def test_stream_compressor_out_of_device_memory(pkg, ctx, monkeypatch):
    import torch
    total = torch.cuda.get_device_properties(ctx.device).total_memory
    monkeypatch.setenv("B200Z_PIPELINE_CHUNK_BYTES", str(total + (1 << 30)))
    data = bytes(datagen.gen_text(3 * (1 << 20) + 5, 41))
    fc = pkg.FrameCompressor(ctx)
    src, sink = Source(data), Sink()
    fc.set_source(src)
    fc.set_drain(sink)
    before = ctx.kernel_launches()
    with pytest.raises(pkg.B200ZError) as e:
        fc.compress()
    assert e.value.code == _err(pkg, "OUT_OF_MEMORY"), e.value
    assert src.calls == 0 and sink.calls == 0 and ctx.kernel_launches() == before
    monkeypatch.delenv("B200Z_PIPELINE_CHUNK_BYTES")
    frame, _ = run(pkg.FrameCompressor(ctx), data)
    check_fastest(pkg, data, frame, pkg.compress_to_vec(ctx, data))
