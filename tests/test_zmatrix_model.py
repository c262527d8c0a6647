"""The libzstd matrix (tests/zmatrix.py) on the CPU: every frame decodes to its input with the oracle and with libzstd, the
256 MiB-window frame is refused at the default window limit, the multi-frame buffers decode whole, and the census of what the
frames hold meets the written floor."""
import pytest

import datagen as G
import zmatrix as Z

# Frames where ruzstd's semantics differ from libzstd's: {frame id: (oracle error leaf, stage)}.  None in this matrix: every frame
# libzstd writes here decodes under ruzstd's rules too.
DEVIATIONS = {}


@pytest.fixture(scope="module")
def frames():
    return Z.frames()


def _libzstd(f):
    d = {"formatted": Z.trained_dict(), "raw": Z.raw_dict_content()}.get(f.dict)
    wl = int(f.window).bit_length() - 1 if f.max_window else None
    return G.decompress(f.data, len(f.plain), raw_dict=d, window_log_max=wl)


def test_every_frame_decodes(oracle, frames):
    assert len(frames) > 300 and sum(len(f.plain) for f in frames) > 100 * Z.MiB
    assert sum(1 for f in frames if len(f.plain) >= Z.MiB and not f.checksum) == 1   # only nochecksum-records
    names = oracle.error_names()
    for f in frames:
        assert _libzstd(f) == f.plain, f.id
        assert Z.headers(f.data)[0]["checksum"] == f.checksum, f.id
        try:
            out, d, _, _, _ = Z.trace(oracle, f)
            err = None
        except oracle.OracleError as e:
            out, err = None, (names[e.code], e.stage)
        if f.id in DEVIATIONS:
            assert err == DEVIATIONS[f.id], (f.id, err)
            continue
        assert err is None, (f.id, err)
        assert out == f.plain, f.id
        assert d.bytes_read_from_source() == len(f.data), f.id
        if d.get_checksum_from_data() is not None:
            assert d.get_checksum_from_data() == d.get_calculated_checksum(), f.id
    assert set(DEVIATIONS) <= {f.id for f in frames}


def test_window_log_28_frame(oracle, frames):
    f = Z.by_id(frames)["wlog28-stream-256MiB-window"]
    assert f.window == 256 * Z.MiB and f.max_window == Z.RAISED_MAX_WINDOW
    with pytest.raises(oracle.OracleError) as e:
        Z.oracle_decoder(oracle, f, max_window=Z.DEFAULT_MAX_WINDOW)
    assert oracle.error_names()[e.value.code] == "ZO_ERR_WINDOW_SIZE_TOO_BIG"
    d, r = Z.oracle_decoder(oracle, f)
    d.decode_blocks(r, oracle.ALL)
    assert d.collect() == f.plain


def test_multi_frame_buffers(oracle, frames):
    for name, (buf, plain, ids) in Z.multi_frame_buffers(frames).items():
        assert oracle.FrameDecoder().decode_all(buf, len(plain)) == plain, name
        assert G.decompress(buf, len(plain)) == plain, name


def test_census_meets_floor(oracle, frames):
    c, exact = Z.census(oracle, frames)
    print("\n" + Z.format_census(c))
    for k, why in sorted(Z.UNREACHABLE.items()):
        print(f"not reached: {k}: {why}")
    short = {k: c[k] for k, v in Z.FLOOR.items() if c[k] < v and k not in Z.UNREACHABLE}
    assert not short, f"the census is below the floor: {short}"
    reached = [k for k in Z.UNREACHABLE if c[k] >= Z.FLOOR[k]]
    assert not reached, f"now reached by the matrix, so no longer to be excused: {reached}"
    assert set(Z.UNREACHABLE) <= set(Z.FLOOR)
    assert sum(map(sum, exact.values())) == c["exact-path blocks"]
    # the shapes the matrix is named after
    assert c["largest offset"] > 20 * Z.MiB and c["most blocks in a frame"] >= 500 and c["window_log 28"] == 1
