"""k_huf's bit-reader rings on the GPU: the crafted literal sections at the narrow ring's edges (tests/hufring.py) decode exactly
like the other crafted entropy sections (tests/test_gpu_entropy.py), with both execution kernels and through both rings (the wide
one in small submissions, the narrow one in a submission padded into the band where it saves the second wave); and k_huf and
k_fse each take one wave for a 1 GiB submission of 128 KiB blocks, so that no second wave of serial Huffman or FSE chains doubles
their time."""
import numpy as np
import pytest

import datagen
import entcraft as E
import hufring as H
from test_gpu_entropy import _run

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["cta", "warp"])
def exec_mode(request, monkeypatch):
    monkeypatch.setenv("B200Z_EXEC_MODE", request.param)
    return request.param


@pytest.fixture
def checksummed(pkg, ctx):
    old = ctx.L.b200z_ctx_flags(ctx.h)
    ctx.set_flags(old | pkg.binding.FLAG_CHECKSUM)
    yield
    ctx.set_flags(old)


def test_ring_edges_one_batch(pkg, ctx, exec_mode, checksummed):
    _run(pkg, ctx, H.cases())


def test_ring_edges_one_frame_per_submission(pkg, ctx, exec_mode, checksummed):
    for c in H.cases():
        _run(pkg, ctx, [c])


def test_ring_edges_narrow_ring(pkg, ctx, exec_mode, checksummed):
    """The same cases in a submission padded with Raw blocks to just more than one wave of the wide ring: k_huf takes the narrow
    ring there, and only there."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    b = _batch_of_blocks(pkg, ctx, 8)
    wide = b.debug_waves()["k_huf_ctas_per_sm"]
    b.close()
    nblocks = wide * sms * 8 + 1
    b = _batch_of_blocks(pkg, ctx, nblocks)
    w = b.debug_waves()
    b.close()
    assert w["k_huf"] == 1 and w["k_huf_ctas_per_sm"] > wide, w
    cs = H.cases()
    filler = E.Case("filler", "raw-block", [("raw", b"filler!!")])
    _run(pkg, ctx, cs + [filler] * (nblocks - len(cs)))


def _batch_of_blocks(pkg, ctx, nblocks):
    """A batch of nblocks single-block frames (the waves depend on the block count only)."""
    f = datagen.compress(b"waves " * 40)
    comp = np.frombuffer(f * nblocks, dtype=np.uint8)
    io = np.zeros(nblocks, dtype=pkg.binding.FRAME_IO_DTYPE)
    io["src_off"] = np.arange(nblocks) * len(f)
    io["src_size"] = len(f)
    io["out_off"] = np.arange(nblocks) * 240
    io["out_cap"] = 240
    return pkg.Batch(ctx, comp, io)


def test_entropy_kernels_take_one_wave_at_8192_blocks(pkg, ctx):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms < 132:
        pytest.skip(f"{sms} SMs: the one-wave bound is for 132 or more")

    def waves(nblocks):
        b = _batch_of_blocks(pkg, ctx, nblocks)
        w = b.debug_waves()
        b.close()
        return w

    w = waves(8192)
    assert w["k_huf"] == 1 and w["k_fse"] == 1, w
    narrow = w["k_huf_ctas_per_sm"]
    # a submission that fits in one wave of the wide ring keeps the wide ring (fewer CTAs per SM, faster chains)
    small = waves(8)
    wide = small["k_huf_ctas_per_sm"]
    assert small["k_huf"] == 1 and 0 < wide < narrow, (small, w)
    at_wide = waves(wide * sms * 8)
    assert at_wide["k_huf"] == 1 and at_wide["k_huf_ctas_per_sm"] == wide, at_wide
    # one more block than the narrow ring holds at once needs a second wave with either ring: the wide ring again
    over = waves(narrow * sms * 8 + 1)
    assert over["k_huf"] == 2 and over["k_huf_ctas_per_sm"] == wide, over
