"""CPU oracle for the island tracks of glom_b200_island_track (csrc/island_track.cu)  --  TEST INFRASTRUCTURE, NOT
PRODUCT CODE.

A numpy restatement of the definition in include/glom_b200_track.h, one (sequence, level) and one time step at a time.
`track` takes any label maps: the kernel's own, so that every output can be compared bit for bit, or garbage ones,
which it skips by the same member rule as the kernels (`tree_oracle.members`).  Only tests/ may import it."""
import numpy as np

from tree_oracle import members


def _best(a, b, counts, n):
    """Pairs (a, b) with their counts -> (n,) best b per a: the largest count, then the smallest b; -1 where a has no
    pair.  And the count of that pair (0 where none)."""
    best = np.full(n, -1, np.int64)
    cnt = np.zeros(n, np.int64)
    if a.size:
        order = np.lexsort((b, -counts, a))                              # per a: largest count, then smallest b
        first = order[np.r_[True, a[order][1:] != a[order][:-1]]]
        best[a[first]] = b[first]
        cnt[a[first]] = counts[first]
    return best, cnt


def track(labels, time_dim=0):
    """labels (..., L, n) int with leading dimension `time_dim` as time (the layout of ``islands(states).labels``) ->
    dict of prev, overlap, next, track int32 in the same shape."""
    labels = np.asarray(labels)
    lead = labels.shape[:-2]
    L, n = labels.shape[-2:]
    lab = np.moveaxis(labels, time_dim, 0)
    moved = lab.shape
    T = moved[0]
    lab = lab.reshape(T, -1, L, n)
    S = lab.shape[1]
    prev = np.full((T, S, L, n), -1, np.int64)
    overlap = np.zeros((T, S, L, n), np.int64)
    nxt = np.full((T, S, L, n), -1, np.int64)
    trk = np.full((T, S, L, n), -1, np.int64)
    for s in range(S):
        for l in range(L):
            m = [members(lab[t, s, l]) for t in range(T)]
            for t in range(1, T):
                both = (m[t] >= 0) & (m[t - 1] >= 0)
                keys, counts = np.unique(m[t][both] * n + m[t - 1][both], return_counts=True)
                j, k = keys // n, keys % n
                prev[t, s, l], overlap[t, s, l] = _best(j, k, counts, n)
                nxt[t - 1, s, l] = _best(k, j, counts, n)[0]
            for t in range(T):
                ids = np.full(n, -1, np.int64)
                j = np.flatnonzero(m[t] == np.arange(n))                     # the roots
                k = prev[t, s, l, j]
                mutual = (k >= 0) & (nxt[t - 1, s, l, np.maximum(k, 0)] == j) if t > 0 else np.zeros(j.size, bool)
                ids[j] = np.where(mutual, trk[t - 1, s, l, np.maximum(k, 0)], t * n + j)
                ok = m[t] >= 0
                trk[t, s, l, ok] = ids[m[t][ok]]

    def back(a):
        return np.moveaxis(a.reshape(moved), 0, time_dim).astype(np.int32).reshape(*lead, L, n)
    return dict(prev=back(prev), overlap=back(overlap), next=back(nxt), track=back(trk))
