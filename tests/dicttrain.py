"""A plain NumPy model of the raw-content dictionary trainer (DESIGN.md section 4.5), written from the algorithm's statement and
calling nothing in the library.  The GPU trainer (b200z_dict_train_raw) must give the same dictionary and segment table byte for
byte.

    train(data, dict_size, sample_sizes=None, segment_size=2048) -> (dictionary bytes, [(epoch, src_off, size, score), ...])

The segment list is in epoch order.
"""
import numpy as np

K = 16
F = 22
P1 = np.uint64(0x9E3779B185EBCA87)
P2 = np.uint64(0xC2B2AE3D27D4EB4F)
NO_SLOT = np.uint32(0xFFFFFFFF)
MIN_EPOCH = 10000


def epoch_info(n, dict_size, seg):
    """(number of epochs E, epoch size es, L): compute_epoch_info with n bytes in place of the number of k-mers."""
    L = min(seg, n)
    E = max(1, dict_size // L)
    es = n // E
    if es < MIN_EPOCH:
        es = min(MIN_EPOCH, n)
        E = n // es
    return E, es, L


def epochs(n, dict_size, seg):
    """[(e0, e1, L_e)] for every epoch; the last one runs to n."""
    E, es, L = epoch_info(n, dict_size, seg)
    out = []
    for e in range(E):
        e0, e1 = e * es, (n if e == E - 1 else (e + 1) * es)
        out.append((e0, e1, min(L, e1 - e0)))
    return out


def slots(data, sample_sizes=None):
    """slot(p) of every position p (NO_SLOT where the 16 bytes from p leave p's sample)."""
    a = np.frombuffer(bytes(data), dtype=np.uint8)
    n = a.size
    out = np.full(n, NO_SLOT, dtype=np.uint32)
    if n < K:
        return out
    m = n - K + 1
    w = np.zeros((m, 16), dtype=np.uint8)
    for j in range(16):
        w[:, j] = a[j:j + m]
    lo = w[:, :8].copy().view("<u8").ravel()
    hi = w[:, 8:].copy().view("<u8").ravel()
    with np.errstate(over="ignore"):
        b = hi * P2
        rot = (b << np.uint64(31)) | (b >> np.uint64(33))
        h = ((lo * P1) ^ rot) * P1
    out[:m] = (h >> np.uint64(64 - F)).astype(np.uint32)
    sizes = [n] if sample_sizes is None else [int(s) for s in sample_sizes]
    end = 0
    for s in sizes:
        end += s
        out[max(end - s, end - K + 1, 0):end] = NO_SLOT
    return out


def prev_distance(sl, W):
    """Distance from p back to the nearest earlier position with the same slot when it is at most W - 1 away, else 0."""
    n = sl.size
    d = np.zeros(n, dtype=np.int64)
    pos = np.nonzero(sl != NO_SLOT)[0]
    if pos.size < 2:
        return d
    order = pos[np.argsort(sl[pos], kind="stable")]
    same = sl[order[1:]] == sl[order[:-1]]
    gap = order[1:] - order[:-1]
    ok = same & (gap <= W - 1)
    d[order[1:][ok]] = gap[ok]
    return d


def train(data, dict_size, sample_sizes=None, segment_size=2048):
    data = bytes(data)
    n = len(data)
    if sample_sizes is not None:
        assert sum(int(s) for s in sample_sizes) == n
    assert 16 <= segment_size <= 65536
    if n < K:
        return data, []
    if dict_size == 0:
        return b"", []
    sl = slots(data, sample_sizes)
    freq = np.bincount(sl[sl != NO_SLOT], minlength=1 << F).astype(np.int64)
    W = min(segment_size, n) - K + 1
    dist = prev_distance(sl, W)
    segs = []
    for e, (e0, e1, Le) in enumerate(epochs(n, dict_size, segment_size)):
        We = Le - K + 1
        smax = e1 - Le
        p = np.arange(e0, e1 - K + 1)
        s = sl[e0:e1 - K + 1]
        d = dist[e0:e1 - K + 1]
        has = s != NO_SLOT
        p, s, d = p[has], s[has], d[has]
        lo = np.maximum(p - We + 1, e0)
        prev_ok = (d > 0) & (d <= We - 1) & (p - d >= e0)
        lo = np.where(prev_ok, np.maximum(lo, p - d + 1), lo)
        hi = np.minimum(p, smax)
        f = freq[s]
        use = (lo <= hi) & (f > 0)
        diff = np.zeros(smax - e0 + 2, dtype=np.int64)
        np.add.at(diff, lo[use] - e0, f[use])
        np.add.at(diff, hi[use] - e0 + 1, -f[use])
        score = np.cumsum(diff[:-1])
        best = int(np.argmax(score))          # the first of the largest: the smallest start wins a tie
        start = e0 + best
        segs.append((e, start, Le, int(score[best])))
        chosen = sl[start:start + We]
        freq[chosen[chosen != NO_SLOT]] = 0
    order = sorted(segs, key=lambda t: (t[3], t[0]))
    out = b"".join(data[st:st + sz] for _, st, sz, _ in order)
    return out[max(0, len(out) - dict_size):], segs
