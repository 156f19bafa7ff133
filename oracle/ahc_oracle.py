"""Oracle for agglomerative clustering and the diarization assembly (tests only; numpy fp64, no GPU).

  * ``naive_ahc``: the sequential algorithm, O(N^3): at every step the live pair of least distance in (d, lower
    representative, higher representative) order merges (a cluster's representative is its smallest point), with the
    engine's update formula, until ``stop_k`` clusters are left or the next height exceeds ``stop_height``.
  * ``replay``: checks a linkage matrix against the distances without assuming any tie rule.  Rows are replayed in
    order; each must name two live clusters, its height must equal their linkage distance computed from the original
    points (average: the mean over all member pairs; complete: the max) and the least such distance over all live
    pairs, both within ``rtol`` relative, and its size must be the sum of theirs.
  * ``frame_labels_brute`` / ``segments_brute``: the diarization assembly frame by frame.
"""
from __future__ import annotations

import numpy as np


def distances(S):
    """The engine's distances: d = 1 - S (fp64) from the strict upper triangle of S, mirrored, zero diagonal."""
    S = np.asarray(S, np.float32)
    d = 1.0 - S.astype(np.float64)
    d = np.triu(d, 1)
    return d + d.T


def _label_clusters(parent, N):
    lab = np.full(N, -1, np.int32)
    out = np.empty(N, np.int32)
    nxt = 0
    for i in range(N):
        r = i
        while parent[r] != r:
            r = parent[r]
        if lab[r] < 0:
            lab[r] = nxt
            nxt += 1
        out[i] = lab[r]
    return out


def naive_ahc(d, linkage="average", stop_k=1, stop_height=np.inf):
    """(Z (m, 4), labels (N,) int32) of the sequential algorithm on the symmetric fp64 distances d (N, N)."""
    d = np.array(d, np.float64, copy=True)
    N = d.shape[0]
    live = np.ones(N, bool)                 # slot i holds the cluster whose representative is i
    size = np.ones(N, np.int64)
    cid = np.arange(N)
    parent = np.arange(N)
    Z = []
    iu = np.triu_indices(N, 1)
    while live.sum() > stop_k:
        m = live[iu[0]] & live[iu[1]]
        vals = np.where(m, d[iu], np.inf)
        h = vals.min()
        if not h <= stop_height:
            break
        t = int(np.flatnonzero(vals == h)[0])   # triu order = (lower, higher) representative order
        a, b = int(iu[0][t]), int(iu[1][t])
        na, nb = float(size[a]), float(size[b])
        for c in np.flatnonzero(live):
            if c == a or c == b:
                continue
            if linkage == "average":
                nc = float(size[c])
                v = (na * nc * d[a, c] + nb * nc * d[b, c]) / ((na + nb) * nc)
            else:
                v = max(d[a, c], d[b, c])
            d[a, c] = d[c, a] = v
        Z.append([min(cid[a], cid[b]), max(cid[a], cid[b]), h, size[a] + size[b]])
        cid[a] = N + len(Z) - 1
        size[a] += size[b]
        live[b] = False
        parent[b] = a
    return np.array(Z, np.float64).reshape(-1, 4), _label_clusters(parent, N)


def _close(a, b, rtol):
    return abs(a - b) <= rtol * max(abs(a), abs(b), 1e-3)   # heights are distances of order 1


def replay(Z, d, linkage="average", rtol=1e-12):
    """None if Z (m, 4) is a valid run of the linkage on the fp64 distances d (N, N); else a string saying which row
    fails and why."""
    d = np.asarray(d, np.float64)
    N = d.shape[0]
    # cluster-level sums (average) or maxima (complete) over member pairs, from the original points
    agg = d.copy()
    np.fill_diagonal(agg, np.inf)
    size = {i: 1 for i in range(N)}
    slot = {i: i for i in range(N)}          # cluster id -> row of agg
    live = np.ones(N, bool)

    def link(x, y):
        v = agg[x, y]
        return v / (float(np.sum(size_of[x])) * float(np.sum(size_of[y]))) if linkage == "average" else v

    size_of = np.ones(N, np.int64)
    for r, (fa, fb, h, n) in enumerate(np.asarray(Z, np.float64)):
        ia, ib = int(fa), int(fb)
        if ia != fa or ib != fb or ia not in slot or ib not in slot or ia == ib:
            return f"row {r}: ({fa}, {fb}) are not two live clusters"
        x, y = slot[ia], slot[ib]
        if not _close(h, link(x, y), rtol):
            return f"row {r}: height {h!r} != linkage distance {link(x, y)!r}"
        idx = np.flatnonzero(live)
        sub = agg[np.ix_(idx, idx)]
        if linkage == "average":
            sub = sub / np.outer(size_of[idx], size_of[idx]).astype(np.float64)
        best = sub.min()
        if not _close(h, best, rtol):
            return f"row {r}: height {h!r} != least live distance {best!r}"
        if n != size[ia] + size[ib]:
            return f"row {r}: size {n} != {size[ia]} + {size[ib]}"
        # merge y into x
        if linkage == "average":
            agg[x, :] = agg[x, :] + agg[y, :]
        else:
            agg[x, :] = np.maximum(agg[x, :], agg[y, :])
        agg[:, x] = agg[x, :]
        agg[x, x] = np.inf
        agg[y, :] = np.inf
        agg[:, y] = np.inf
        live[y] = False
        size_of[x] += size_of[y]
        new = N + r
        size[new] = size.pop(ia) + size.pop(ib)
        del slot[ia], slot[ib]
        slot[new] = x
    return None


def frame_labels_brute(win_start, win_labels, n_frames, T):
    """Per frame: among the windows [s, s + T) covering it (a recording shorter than T: its one window covers every
    frame), the one whose centre s + T/2 is nearest to f + 1/2, the earlier on a tie."""
    out = np.empty(n_frames, np.int32)
    starts = [int(s) for s in win_start]
    for f in range(n_frames):
        best, bw = None, None
        for w, s in enumerate(starts):
            if not (s <= f < s + T or len(starts) == 1):
                continue
            dist = abs((f + 0.5) - (s + T / 2))
            if best is None or dist < best:
                best, bw = dist, w
        assert bw is not None, f"frame {f} is not covered"
        out[f] = win_labels[bw]
    return out


def segments_brute(labels, frame_shift=0.01):
    out = []
    for f, k in enumerate(labels):
        if out and out[-1][2] == int(k):
            out[-1][1] = (f + 1) * frame_shift
        else:
            out.append([f * frame_shift, (f + 1) * frame_shift, int(k)])
    return [tuple(x) for x in out]
