"""CPU oracle for the part-whole trees of glom_b200_island_tree (csrc/island_tree.cu)  --  TEST INFRASTRUCTURE,
NOT PRODUCT CODE.

The reference has no implementation of the analysis (its README only says the returned states are there "for
clustering, from which one can inspect for the theorized islands"), so this numpy restatement of the definition in
include/glom_b200_tree.h is the only checker.  `tree` takes any label maps: the kernel's own, so that the integer outputs
can be compared bit for bit, or garbage ones, which it skips by the same member rule as the kernels.  Only tests/ may
import it."""
import numpy as np


def members(lab):
    """lab (n,) int labels of one level -> (n,) int64: the island each patch is a member of, or -1.  Patch i is a member
    of j = lab[i] when 0 <= j <= i and lab[j] == j (include/glom_b200_tree.h)."""
    lab = np.asarray(lab).astype(np.int64)
    idx = np.arange(lab.shape[0])
    ok = (lab >= 0) & (lab <= idx)
    j = np.where(ok, lab, 0)
    return np.where(ok & (lab[j] == j), lab, -1)


def tree(labels, states=None):
    """labels (..., L, n) int32 -> dict of size, parent int32 (..., L, n), containment float32 (..., L, n), nested
    float32 (..., L-1); with states (..., n, L, d) also embedding (..., L, n, d), member_cos and coherence (..., L, n),
    all float64 (sums in float64).  The integer outputs, containment and nested are what the kernels must give bit for
    bit: containment and nested are one fp32 division of exact integers."""
    labels = np.asarray(labels)
    *lead, L, n = labels.shape
    lab = labels.reshape(-1, L, n)
    S = lab.shape[0]
    size = np.zeros((S, L, n), np.int32)
    parent = np.full((S, L, n), -1, np.int32)
    containment = np.zeros((S, L, n), np.float32)
    nested = np.zeros((S, max(L - 1, 0)), np.float32)
    if states is not None:
        x_all = np.asarray(states).reshape(S, n, L, -1)
        d = x_all.shape[-1]
        emb = np.zeros((S, L, n, d))
        mcos = np.zeros((S, L, n))
        coh = np.zeros((S, L, n))
    for s in range(S):
        m = [members(lab[s, l]) for l in range(L)]
        for l in range(L):
            ok = m[l] >= 0
            size[s, l] = np.bincount(m[l][ok], minlength=n)
            if l + 1 < L:
                both = ok & (m[l + 1] >= 0)
                keys, counts = np.unique(m[l][both] * n + m[l + 1][both], return_counts=True)
                j, k = keys // n, keys % n
                order = np.lexsort((k, -counts, j))                     # per j: largest overlap, then smallest k
                first = order[np.r_[True, j[order][1:] != j[order][:-1]]] if keys.size else order
                parent[s, l, j[first]] = k[first]
                containment[s, l, j[first]] = np.float32(counts[first]) / np.float32(size[s, l, j[first]])
                whole = counts[first] == size[s, l, j[first]]
                nested[s, l] = np.float32(size[s, l, j[first]][whole].sum()) / np.float32(n)
            if states is not None:
                x = x_all[s, :, l, :].astype(np.float64)
                acc = np.zeros((n, d))
                np.add.at(acc, m[l][ok], x[ok])
                roots = size[s, l] > 0
                emb[s, l, roots] = acc[roots] / size[s, l, roots][:, None]
                e = emb[s, l, m[l][ok]]
                den = np.maximum(np.sqrt((x[ok] ** 2).sum(-1)) * np.sqrt((e ** 2).sum(-1)), 1e-12)
                mcos[s, l, ok] = (x[ok] * e).sum(-1) / den
                coh[s, l, roots] = np.bincount(m[l][ok], weights=mcos[s, l, ok], minlength=n)[roots] / size[s, l, roots]
    out = dict(size=size.reshape(*lead, L, n), parent=parent.reshape(*lead, L, n),
               containment=containment.reshape(*lead, L, n), nested=nested.reshape(*lead, max(L - 1, 0)))
    if states is not None:
        out.update(embedding=emb.reshape(*lead, L, n, d), member_cos=mcos.reshape(*lead, L, n),
                   coherence=coh.reshape(*lead, L, n))
    return out
