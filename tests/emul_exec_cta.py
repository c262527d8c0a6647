"""Bit-level model of k_exec_cta's data path (zstd-rs_b200/csrc/exec_cta.cuh), for CPU tests of the LOGIC the kernel
relies on: prefix-form records, the 8-byte ring record, the sequence-end bitmask, the per-64-byte chunk owner table, the
sentinel, "a 4-byte word spans at most two sequences", the literal delta, overlapping matches (k mod offset), sources in
earlier blocks of the frame, in-row dependencies.  Rows are produced in order (the concurrency -- rows-done bitmap,
barriers -- is not modelled).  Test infrastructure only."""
import numpy as np

XC_BATCH = 1024
XC_RING = 2048
XC_WIN_MAX = 128 << 10
XC_DATA_BYTES = 182 << 10
SYM_SHIFT = 30
XC_LITG_BIAS = (1 << 17) + 64


def sym_resolve(v, h):
    tag = v >> SYM_SHIFT
    if tag == 0:
        return v
    d = v & ((1 << SYM_SHIFT) - 1)
    hh = h[tag - 1]
    return hh - d if hh > d else 0


def pack(mstart_a, lz, off):
    lo = (mstart_a | (lz << 18)) & 0xFFFFFFFF
    hi = ((lz >> 14) | (off << 4)) & 0xFFFFFFFF
    return lo, hi


def unpack(lo, hi):
    x = lo & 0x3FFFF
    lz = (((hi << 32) | lo) >> 18) & 0x3FFFF
    noff = -(hi >> 4)
    return x, lz, noff


class Bail(Exception):
    pass


def exec_block(prefix_records, hist, literals, earlier, gaddr, loff=0):
    """prefix_records: (n, 3) uint32 {out_end, lit_end, of_symbolic}; hist: offset history at the block's start;
    literals: bytes; earlier: bytes of the frame produced before this block (all reachable); gaddr: global address of the
    block's first output byte (only its low 4 bits matter).  Returns the block's output bytes."""
    nseq = len(prefix_records)
    regen = len(literals)
    sum_ll = int(prefix_records[-1][1]) if nseq else 0
    out_size = (int(prefix_records[-1][0]) - sum_ll if nseq else 0) + regen
    if out_size > XC_WIN_MAX or sum_ll > regen:
        raise Bail("size")
    if out_size == 0:
        return b""
    woff = gaddr & 15
    a_end = woff + out_size
    wbytes = (a_end + 127) & ~127
    nrows = wbytes >> 7
    ntot = nseq + (1 if regen > sum_ll else 0)
    lit_bytes = (loff + regen + 15) & ~15
    litg = wbytes + lit_bytes > XC_DATA_BYTES      # literals read from "global memory" (the bytes object) byte by byte
    lit_s = wbytes + loff
    reach = len(earlier)
    data = bytearray(XC_DATA_BYTES)
    if not litg:
        data[lit_s:lit_s + regen] = literals
    mask = np.zeros(nrows * 128 + 64, dtype=np.uint8)      # one entry per window byte (the kernel packs them 32 per word)
    first = np.full(nrows * 2, 0xDEADBEEF, dtype=np.int64)
    ring = [(0x12345678, 0x9ABCDEF0)] * XC_RING            # stale garbage
    ovl = [0, 0, 0, 0]
    end_a_of = [0, 0]

    def rec(i):
        if i < nseq:
            return int(prefix_records[i][0]), int(prefix_records[i][1]), int(prefix_records[i][2])
        return out_size, regen, 0

    def build(k):
        for tid in range(XC_BATCH):
            i = k * XC_BATCH + tid
            if i > ntot:
                break
            if i == ntot:
                ring[i & (XC_RING - 1)] = pack(0x3FFFF, 0, 1)
                for c in range((a_end + 63) >> 6, nrows * 2):
                    first[c] = i
                end_a_of[k & 1] = a_end
                continue
            cur_out, cur_lit, of = rec(i)
            p_out, p_lit = (0, 0) if i == 0 else rec(i - 1)[:2]
            real = i < nseq
            ll = cur_lit - p_lit
            start, end = p_out, cur_out
            mstart = start + ll
            ml = end - mstart
            off = sym_resolve(of, hist) if real else 1
            bad = end > out_size or end <= start or mstart > end or cur_lit > regen or cur_lit < p_lit
            if real:
                bad = bad or off == 0 or off >= (1 << 28) or off > reach + mstart or ml < 3
            if bad:
                raise Bail("sequence %d" % i)
            if off < ml:
                ovl[k & 3] = 1
            start_a, end_a = woff + start, woff + end
            lz = (XC_LITG_BIAS if litg else lit_s) + cur_lit - woff - mstart
            assert 0 <= lz < (1 << 18)
            ring[i & (XC_RING - 1)] = pack(woff + mstart, lz, off)
            mask[end_a - 1] = 1
            c_lo = 0 if i == 0 else (start_a + 63) >> 6
            for c in range(c_lo, ((end_a - 1) >> 6) + 1):
                first[c] = i
            if i + 1 == (k + 1) * XC_BATCH:
                end_a_of[k & 1] = end_a

    def row(r, has_ovl):
        row_a = r << 7
        src = np.zeros(128, dtype=np.int64)
        mt = np.zeros(128, dtype=bool)
        for lane in range(32):
            a0 = row_a + 4 * lane
            c = a0 >> 6
            owner0 = int(first[c]) + int(mask[c * 64:a0].sum())
            nib = int(mask[a0]) | (int(mask[a0 + 1]) << 1) | (int(mask[a0 + 2]) << 2)
            A = unpack(*ring[owner0 & (XC_RING - 1)])
            B = unpack(*ring[(owner0 + 1) & (XC_RING - 1)])
            for k in range(4):
                useB = k > 0 and (nib & ((1 << k) - 1)) != 0
                x, lz, noff = B if useB else A
                a = a0 + k
                m = a >= x
                s = a + (noff if m else lz)
                if has_ovl:
                    kk, off = a - x, -noff
                    if m and kk >= off:
                        s = x - off + kk % off
                src[4 * lane + k], mt[4 * lane + k] = s, m
        # gather: everything whose source is outside the row first, then the in-row bytes in rounds
        vals = np.zeros(128, dtype=np.int64)
        pend = np.zeros(128, dtype=bool)
        for j in range(128):
            s = int(src[j])
            if mt[j] and s >= max(row_a, woff):
                pend[j] = True
            elif mt[j] and s < woff:
                g = s - woff                       # relative to the block's first byte: negative
                assert -g <= reach, "far source beyond the reachable output"
                vals[j] = earlier[len(earlier) + g]
            elif litg and not mt[j]:
                vals[j] = literals[min((s - XC_LITG_BIAS) & 0xFFFFFFFF, regen - 1)]
            else:
                assert 0 <= s < XC_DATA_BYTES
                vals[j] = data[s]
        for j in range(128):
            if not pend[j]:
                data[row_a + j] = int(vals[j])
        rounds = 0
        while pend.any():
            snap = pend.copy()
            for j in range(128):
                if snap[j] and not snap[int(src[j]) - row_a]:
                    data[row_a + j] = data[int(src[j])]
                    pend[j] = False
            rounds += 1
            assert rounds <= 128
        return rounds

    nbatch = (ntot + 1 + XC_BATCH - 1) // XC_BATCH
    build(0)
    row_lo = 0
    for k in range(nbatch):
        last = k + 1 == nbatch
        row_hi = nrows if last else end_a_of[k & 1] >> 7
        has_ovl = bool(ovl[k & 3] | ovl[(k + 3) & 3])
        ovl[(k + 2) & 3] = 0
        for r in range(row_lo, row_hi):
            row(r, has_ovl)
        if not last:
            build(k + 1)
        row_lo = row_hi
    return bytes(data[woff:a_end])


def to_prefix(ll, ml, of_sym):
    """(n,) arrays -> the (n, 3) prefix-form records k_fse writes"""
    ll = np.asarray(ll, dtype=np.uint64)
    ml = np.asarray(ml, dtype=np.uint64)
    out_end = np.cumsum(ll + ml)
    lit_end = np.cumsum(ll)
    return np.stack([out_end, lit_end, np.asarray(of_sym, dtype=np.uint64)], axis=1).astype(np.uint32)


def symbolic_offsets(ll, of_raw):
    """do_offset_history (sequence_execution.rs:59-118) on symbolic history values, as k_fse's fse_step does it.
    Returns (of_sym array, hist_after)."""
    h = [1 << SYM_SHIFT, 2 << SYM_SHIFT, 3 << SYM_SHIFT]
    out = []
    for l, of in zip(ll, of_raw):
        l, of = int(l), int(of)
        if of <= 3:
            r = of - 1 + (1 if l == 0 else 0)
            if r == 0:
                actual = h[0]
            elif r == 1:
                actual = h[1]; h[1] = h[0]
            elif r == 2:
                actual = h[2]; h[2] = h[1]; h[1] = h[0]
            else:
                actual = (h[0] + 1) if (h[0] >> SYM_SHIFT) else (h[0] - 1 if h[0] else 0)
                h[2] = h[1]; h[1] = h[0]
            h[0] = actual
        else:
            actual = of - 3
            h[2] = h[1]; h[1] = h[0]; h[0] = actual
        out.append(actual)
    return np.array(out, dtype=np.uint64), h


def run_frame(oracle, data, max_blocks=None, base=0x1005, strict=False):
    """Runs the Compressed blocks of a frame through the model: the oracle's per-block traces ({ll, ml, offset_value},
    literals) are turned into what k_fse hands over -- prefix-form records with symbolic offsets -- and each block's output
    must be the reference's.  base: global address of the frame's first byte.  A block the model bails out of is skipped,
    or fails the check when `strict`.  Returns (blocks run, sequences run)."""
    d = oracle.FrameDecoder(); d.trace_enable()
    r = d.reset(data); d.decode_blocks(r); out = d.collect()
    blocks, lits, seqs = d.trace()
    hist = [1, 4, 8]
    pos = 0
    nblk = nseq = 0
    for tb in blocks:
        size = tb["out_size"]
        if tb["block_type"] == 2:
            n = tb["num_sequences"]
            s = seqs[tb["seq_offset"]:tb["seq_offset"] + n]
            lit = lits[tb["lit_offset"]:tb["lit_offset"] + tb["regenerated_size"]]
            sym, h_after = symbolic_offsets(s[:, 0], s[:, 2])
            # symbols resolve to the reference's actual offsets, and the history carries over symbolically
            got_actual = np.array([sym_resolve(int(v), hist) for v in sym], dtype=np.uint64)
            assert np.array_equal(got_actual, s[:, 3].astype(np.uint64))
            if max_blocks is None or nblk < max_blocks:
                rec = to_prefix(s[:, 0], s[:, 1], sym)
                try:
                    got = exec_block(rec, hist, lit, out[:pos], base + pos)
                    assert got == out[pos:pos + size], (nblk, size)
                except Bail:
                    if strict:
                        raise
                nblk += 1; nseq += n
            if n:
                hist = [sym_resolve(int(v), hist) for v in h_after]
                assert hist == list(tb["offset_hist_after"])
        pos += size
    assert pos == len(out)
    return nblk, nseq
