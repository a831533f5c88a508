"""CPU oracle for the island analytics (csrc/islands.cu)  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The reference has no implementation of the analysis its README describes (README.md:34-36: inspect the returned
states "for the theorized islands"); this numpy restatement of the definition in include/glom_b200.h is therefore the
only checker ("parity unpinned": there is nothing in the reference to pin it on).  Only tests/ may import it.

`edges` gives the neighbour cosine maps, `components` the labels and island count of thresholded maps, and `islands`
composes the two with the agreement map.  `components` takes any maps, so the labels can be checked on the kernel's own
fp32 cosines, without a margin around the threshold."""
import numpy as np


def edges(states, side_h, side_w):
    """states (..., n, L, d) -> (cos_right, cos_down) float64 (..., L, n): cosine similarity of patch (h, w) with
    (h, w + 1) / (h + 1, w), 0 in the last column / row."""
    x = np.asarray(states, dtype=np.float64)
    *lead, n, L, d = x.shape
    assert n == side_h * side_w
    g = np.moveaxis(x, -2, -3).reshape(*lead, L, side_h, side_w, d)          # (..., L, h, w, d)
    nrm = np.sqrt((g * g).sum(-1))
    cr = np.zeros(g.shape[:-1])
    cd = np.zeros(g.shape[:-1])
    cr[..., :, :-1] = (g[..., :, :-1, :] * g[..., :, 1:, :]).sum(-1) / np.maximum(nrm[..., :, :-1] * nrm[..., :, 1:], 1e-12)
    cd[..., :-1, :] = (g[..., :-1, :, :] * g[..., 1:, :, :]).sum(-1) / np.maximum(nrm[..., :-1, :] * nrm[..., 1:, :], 1e-12)
    shp = (*lead, L, n)
    return cr.reshape(shp), cd.reshape(shp)


def components(cos_right, cos_down, side_h, side_w, threshold):
    """Maps (..., L, n) -> (labels int32 (..., L, n), num_islands int32 (..., L)): the 4-connected components of the
    neighbour pairs with cosine >= threshold, each labelled by its smallest patch index.  The comparison is done in the
    maps' own dtype."""
    cr, cd = np.asarray(cos_right), np.asarray(cos_down)
    shp = cr.shape
    n = side_h * side_w
    assert shp[-1] == n and cd.shape == shp
    flat_r = cr.reshape(-1, side_h, side_w)
    flat_d = cd.reshape(-1, side_h, side_w)
    labels = np.empty((flat_r.shape[0], n), dtype=np.int32)
    counts = np.empty(flat_r.shape[0], dtype=np.int32)
    for k in range(flat_r.shape[0]):                                  # union-find per (slab, level)
        keep_r = flat_r[k] >= threshold
        keep_d = flat_d[k] >= threshold
        parent = list(range(n))

        def find(a):
            while parent[a] != a:
                parent[a] = parent[parent[a]]
                a = parent[a]
            return a
        for h in range(side_h):
            for w in range(side_w):
                i = h * side_w + w
                if w + 1 < side_w and keep_r[h, w]:
                    a, b = find(i), find(i + 1)
                    parent[max(a, b)] = min(a, b)
                if h + 1 < side_h and keep_d[h, w]:
                    a, b = find(i), find(i + side_w)
                    parent[max(a, b)] = min(a, b)
        roots = [find(i) for i in range(n)]
        labels[k] = roots
        counts[k] = len(set(roots))
    return labels.reshape(shp), counts.reshape(shp[:-1])


def islands(states, side_h, side_w, threshold):
    """states (..., n, L, d) -> dict of cos_right, cos_down, agreement (..., L, n), labels int32, num_islands (..., L)."""
    cr, cd = edges(states, side_h, side_w)
    shp = cr.shape
    gr = cr.reshape(*shp[:-1], side_h, side_w)
    gd = cd.reshape(*shp[:-1], side_h, side_w)
    s = np.zeros_like(gr)
    c = np.zeros_like(gr)
    s[..., :, :-1] += gr[..., :, :-1]; c[..., :, :-1] += 1          # right neighbour
    s[..., :, 1:] += gr[..., :, :-1]; c[..., :, 1:] += 1            # left neighbour
    s[..., :-1, :] += gd[..., :-1, :]; c[..., :-1, :] += 1          # lower neighbour
    s[..., 1:, :] += gd[..., :-1, :]; c[..., 1:, :] += 1            # upper neighbour
    agreement = np.where(c > 0, s / np.maximum(c, 1), 1.0)
    labels, counts = components(cr, cd, side_h, side_w, threshold)
    return dict(cos_right=cr, cos_down=cd, agreement=agreement.reshape(shp), labels=labels, num_islands=counts)
