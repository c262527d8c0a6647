"""decode_all_stream (tier 1d) on the stream case set (tests/streamcraft.py): every crafted decoder case and every stream-edge
family, at chunk sizes that cut each frame at every block boundary and at none, with the checksum flag off and on, with both
execution kernels.  The plaintext must be the oracle's decode_all byte for byte, the summary decode_all_batch's on the same bytes,
the submissions those of the cut model (so the GPU ran the cuts tests/test_streamcraft.py checks), every checksum counted and
matched, and a flipped checksum reported at exactly its frame.  Error cases run one per call after a valid head, and the drain
must hold what the oracle's FrameDecoder delivers before the failing block."""
import collections

import pytest

import dictcraft as D
import streamcraft as SC
import streamcut
from test_gpu_decode_all_stream import SUMMARY, batch, oracle_delivered, stream

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["cta", "warp"])
def exec_mode(request, monkeypatch):
    monkeypatch.setenv("B200Z_EXEC_MODE", request.param)
    return request.param


@pytest.fixture(scope="module")
def cases():
    crafted = SC.crafted()
    every = crafted + SC.new_cases(crafted)
    valid = collections.OrderedDict()
    for c in every:
        if c.valid and not SC.deviation(c):
            valid.setdefault((c.group, c.dicts, c.forced.name if c.forced else None), []).append(c)
    errors = [c for c in every if not c.valid and not SC.deviation(c)]
    return valid, errors


@pytest.fixture(scope="module")
def handles(pkg, ctx, cases):
    """Per dictionary set: (the Dictionary handles, {dictcraft name: handle} for forced dictionaries)."""
    dc = {d.name: (pkg.Dictionary.decode_dict(ctx, d.raw) if d.formatted else pkg.Dictionary.raw_content(ctx, d.id, d.content)) for d in D.DICTS}
    raws = sorted({c.dict_raw for cs in cases[0].values() for c in cs if c.dict_raw is not None} |
                  {c.dict_raw for c in cases[1] if c.dict_raw is not None})
    return {"dictcraft": (list(dc.values()), dc), "entcraft": ([pkg.Dictionary.decode_dict(ctx, r) for r in raws], {}), None: (None, {})}, raws


@pytest.fixture
def flags(ctx):
    old = ctx.L.b200z_ctx_flags(ctx.h)
    yield old
    ctx.set_flags(old)


def _oracle_decoder(oracle, dicts, raws):
    d = D.oracle_decoder(oracle) if dicts == "dictcraft" else oracle.FrameDecoder()
    if dicts == "entcraft":
        for r in raws:
            d.add_dict(r)
    return d


def _frames(at):
    """Per case, its zstd frame index in the stream, and how many zstd frames carry a checksum."""
    idx, n, ck = [], 0, 0
    for c, _, lead, _ in at:
        if lead:
            n, ck = n + 1, ck + 1
        idx.append(n)
        n, ck = n + 1, ck + (1 if c.checksum else 0)
    return idx, ck


def test_valid_streams(pkg, ctx, oracle, cases, handles, exec_mode, monkeypatch, flags):
    hs, raws = handles
    for key, cs in cases[0].items():
        group, dicts, forced = key
        named, by_name = hs[dicts]
        kw = dict(dicts=named, forced_dict=by_name[forced] if forced else None)
        for chunk in SC.CHUNKS:
            data, plain, at = SC.stream(cs, chunk)
            nsub = len(streamcut.cut(SC.stream(cs, chunk, for_cut=True)[0], chunk)[0])
            if forced is None:
                assert _oracle_decoder(oracle, dicts, raws).decode_all(data, len(plain)) == plain, (key, chunk)
            want = batch(pkg, ctx, data, len(plain), **kw)
            idx, nck = _frames(at)
            for flag in (0, 1):
                ctx.set_flags(flags | flag)
                r, out = stream(pkg, ctx, monkeypatch, data, chunk, **kw)
                assert {k: r[k] for k in SUMMARY} == want, (key, chunk, flag)
                assert r["status"] == 0 and r["frames"] == len(idx) + sum(1 for _, _, lead, _ in at if lead), (key, chunk, r)
                if out != plain:
                    bad = next(i for i in range(min(len(out), len(plain))) if out[i] != plain[i]) if out[:len(plain)] != plain[:len(out)] else min(len(out), len(plain))
                    pos = 0
                    for c, _, _, lp in at:
                        if pos + len(lp) + len(c.expected) > bad:
                            break
                        pos += len(lp) + len(c.expected)
                    pytest.fail(f"{key} chunk {chunk} flag {flag}: output differs at byte {bad}, in case {c.id} (byte {bad - pos - len(lp)} of it)")
                assert r["submissions"] == nsub, (key, chunk, r["submissions"], nsub)
                if flag:
                    assert r["checksum_frames"] == nck and r["checksum_mismatches"] == 0, (key, chunk, r)
            # one case's checksum flipped: reported at exactly its frame, the output unchanged
            k = len(cs) // 2
            c, pos, _, _ = at[k]
            end = pos + len(c.frame)
            flipped = data[:end - 4] + bytes(b ^ 0xFF for b in data[end - 4:end]) + data[end:]
            ctx.set_flags(flags | 1)
            r, out = stream(pkg, ctx, monkeypatch, flipped, chunk, **kw)
            assert r["status"] == 0 and out == plain, (key, chunk, c)
            assert r["checksum_mismatches"] == 1 and r["first_mismatch_frame"] == idx[k], (key, chunk, c, r)


def _delivered(oracle, data, r, dicts, raws):
    """oracle_delivered with the dictionaries of the case's set."""
    if dicts is None:
        return oracle_delivered(oracle, data, r)
    if r["status"] == 0 or r["error_frame"] < 0:
        return r["written"]
    d = _oracle_decoder(oracle, dicts, raws)
    d.trace_enable()
    try:
        rd = d.reset(data[r["error_offset"]:])
        while not d.is_finished():
            d.decode_blocks(rd, oracle.UPTO_BLOCKS, 1)
    except oracle.OracleError:
        pass
    return r["written"] + sum(b["out_size"] for b in d.trace()[0][:d.blocks_decoded()])


def test_error_cases(pkg, ctx, oracle, cases, handles, exec_mode, monkeypatch, flags):
    hs, raws = handles
    head_case = cases[0][("carry-tables", None, None)][0]
    head, head_plain = head_case.frame, head_case.expected
    names = pkg.error_names()
    for c in cases[1]:
        named, by_name = hs[c.dicts]
        kw = dict(dicts=named, forced_dict=by_name[c.forced.name] if c.forced else None)
        for chunk in SC.CHUNKS:
            data, _, at = SC.stream([c], chunk, head=head)
            lead_plain = at[0][3]
            cap = len(head_plain) + len(lead_plain) + sum(c.sizes) + 64
            want = batch(pkg, ctx, data, cap, **kw)
            for flag in (0, 1):
                ctx.set_flags(flags | flag)
                r, out = stream(pkg, ctx, monkeypatch, data, chunk, **kw)
                assert {k: r[k] for k in SUMMARY} == want, (c, chunk, flag, r)
                assert r["status"] != 0 and r["error_frame"] == (2 if at[0][2] else 1), (c, chunk, r, names.get(r["status"]))
                assert out.startswith(head_plain + lead_plain), (c, chunk)
                assert len(out) == _delivered(oracle, data, r, c.dicts, raws), (c, chunk, r)
