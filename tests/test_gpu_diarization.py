"""Diarization on the GPU: dsk_ahc against scipy's linkage on the same fp64 distances (bit-exact for complete
linkage, ids and sizes exact and heights within 1e-12 for average), early stops against fcluster, a chain that needs
one round per merge, tie-heavy input through the replay validator, invariances, and diarize end to end against a host
recomposition and against the fp64 pipeline."""
import numpy as np
import pytest
import torch
from scipy.cluster.hierarchy import fcluster
from scipy.cluster.hierarchy import linkage as scipy_linkage
from scipy.optimize import linear_sum_assignment
from scipy.spatial.distance import squareform

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import diarization as DZ
from deepspeaker_pytorch_b200 import engine as EN
from deepspeaker_pytorch_b200 import frontend as F
from oracle import ahc_oracle as O
from oracle import rescnn_oracle as RO

pytestmark = pytest.mark.gpu


def _sims(N, seed, kind):
    rng = np.random.default_rng(seed)
    if kind == "clustered":
        C = rng.standard_normal((8, 64))
        X = C[rng.integers(0, 8, N)] + 0.7 * rng.standard_normal((N, 64))
    else:
        X = rng.standard_normal((N, 64))
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    return (X @ X.T).astype(np.float32)


def _scipy(S, method):
    return scipy_linkage(squareform(O.distances(S), checks=False), method=method)


def _clusters(Z):
    """{(hash of one merged cluster, hash of the other): (height, size)} with a cluster's hash the wrapping sum of
    random 64-bit keys of its points: the tree as a set of merges, whatever the order of rows of equal height."""
    N = Z.shape[0] + 1
    key = list(np.random.default_rng(0).integers(0, 2 ** 63, N, dtype=np.uint64))
    out = {}
    with np.errstate(over="ignore"):
        for a, b, h, n in Z:
            ka, kb = key[int(a)], key[int(b)]
            out[(min(ka, kb), max(ka, kb))] = (h, n)
            key.append(ka + kb)
    return out


def _check_tree(Z, Zs, method):
    """Bit-identical to scipy (average: ids and sizes, heights within 1e-12) when scipy's heights are distinct.  fp32
    cosines of thousands of points can repeat a value, and then rows of equal height may come in either order (the
    engine sorts them by round and representative): the same merges at the same heights are required instead."""
    assert Z.shape == Zs.shape
    if np.unique(Zs[:, 2]).size == Zs.shape[0]:
        if method == "complete":
            assert np.array_equal(Z, Zs)
        else:
            assert np.array_equal(Z[:, [0, 1, 3]], Zs[:, [0, 1, 3]])
            np.testing.assert_allclose(Z[:, 2], Zs[:, 2], rtol=1e-12, atol=0)
        return
    c, cs = _clusters(Z), _clusters(Zs)
    assert c.keys() == cs.keys()
    h, hs = (np.array([m[k] for k in sorted(cs)]) for m in (c, cs))
    assert np.array_equal(h[:, 1], hs[:, 1])
    if method == "complete":
        assert np.array_equal(h[:, 0], hs[:, 0])
    else:
        np.testing.assert_allclose(h[:, 0], hs[:, 0], rtol=1e-12, atol=0)
    print(f"\n{Zs.shape[0] - np.unique(Zs[:, 2]).size} tied heights: compared as sets of merges")


def _relabel(lab):
    """Flat clusters numbered by their smallest member (the engine's numbering)."""
    lab = np.asarray(lab)
    _, first = np.unique(lab, return_index=True)
    order = np.argsort(first)
    remap = np.empty(order.size, np.int64)
    remap[order] = np.arange(order.size)
    return remap[np.searchsorted(np.unique(lab), lab)].astype(np.int32)


@pytest.mark.parametrize("N", [2, 3, 257, 2000, 12000])
@pytest.mark.parametrize("kind", ["random", "clustered"])
def test_ahc_matches_scipy(cuda_dev, N, kind):
    if N == 12000 and kind == "random":
        pytest.skip("one 12 000-point case (clustered) keeps the host side of the suite short")
    S = _sims(N, N, kind)
    Sd = torch.from_numpy(S).to(cuda_dev)
    for method in ("complete", "average"):
        Z, lab, rounds = EN.ahc(Sd, method, return_rounds=True)
        _check_tree(Z, _scipy(S, method), method)
        assert lab.is_cuda and lab.dtype == torch.int32 and torch.all(lab == 0)
        print(f"\nN {N} {kind} {method}: {rounds} rounds")


def test_early_stops_match_fcluster(cuda_dev):
    N = 2000
    S = _sims(N, 5, "clustered")
    Sd = torch.from_numpy(S).to(cuda_dev)
    for method in ("average", "complete"):
        Zf, _ = EN.ahc(Sd, method)
        for k in (1, 2, 8, 50, 1999, 2000):
            Z, lab = EN.ahc(Sd, method, num_clusters=k)
            assert Z.shape[0] == N - k and np.array_equal(Z, Zf[:N - k]), (method, k)
            assert np.array_equal(lab.cpu().numpy(), _relabel(fcluster(Zf, k, "maxclust"))), (method, k)
        for t in (0.3, 0.8, float(Zf[1000, 2]), 1.5, 3.0):
            Z, lab = EN.ahc(Sd, method, threshold=t)
            m = int(np.sum(Zf[:, 2] <= t))
            assert np.array_equal(Z, Zf[:m]), (method, t)
            assert np.array_equal(lab.cpu().numpy(), _relabel(fcluster(Zf, t, "distance"))), (method, t)


def chain_similarities(N):
    """A chain that allows one merge per round: d(i, j) = (j (N + 1) - i) 2^-24 for i < j.  The cluster of points
    0..k-1 and point k are each other's nearest; every later point j is nearest to j - 1, whose own nearest lies
    further left, so each round has exactly one mutual pair and the tree takes N - 1 rounds.  Every distance is
    distinct and below 2, and S = 1 - d is exact in fp32."""
    j = np.arange(N, dtype=np.int64)
    d = np.maximum(j[None, :], j[:, None]) * (N + 1) - np.minimum(j[None, :], j[:, None])
    return (1.0 - d * 2.0 ** -24).astype(np.float32)


def test_chain_needs_one_round_per_merge(cuda_dev):
    N = 3000
    S = chain_similarities(N)
    Sd = torch.from_numpy(S).to(cuda_dev)
    for method in ("complete", "average"):
        Z, _, rounds = EN.ahc(Sd, method, return_rounds=True)
        _check_tree(Z, _scipy(S, method), method)
        print(f"\nchain N {N} {method}: {rounds} rounds for {N - 1} merges")
        assert rounds == N - 1


def _tie_heavy(seed):
    rng = np.random.default_rng(seed)
    S = np.round(rng.uniform(-1, 1, (300, 300)) * 8) / 8          # similarities quantised to 1/8
    S = np.triu(S, 1) + np.triu(S, 1).T
    S[100:200] = S[0:100]                                          # duplicated rows (and columns)
    S[:, 100:200] = S[:, 0:100]
    S[np.arange(100), np.arange(100, 200)] = 1.0
    return [S.astype(np.float32), np.full((257, 257), 0.375, np.float32)]


def test_tie_heavy_replays_and_repeats(cuda_dev):
    for S in _tie_heavy(3):
        Sd = torch.from_numpy(S).to(cuda_dev)
        d = O.distances(S)
        for method in ("average", "complete"):
            Z1, l1 = EN.ahc(Sd, method)
            Z2, l2 = EN.ahc(Sd, method)
            assert Z1.shape == (S.shape[0] - 1, 4)
            assert np.array_equal(Z1, Z2) and torch.equal(l1, l2)
            msg = O.replay(Z1, d, method)
            assert msg is None, (method, msg)


def test_invariances(cuda_dev):
    N = 700
    S = _sims(N, 9, "clustered")
    Sd = torch.from_numpy(S).to(cuda_dev)
    ref = {m: EN.ahc(Sd, m, num_clusters=5) for m in ("average", "complete")}
    g = torch.Generator(device=cuda_dev).manual_seed(1)
    junk = Sd.clone()
    low = torch.ones(N, N, dtype=torch.bool, device=cuda_dev).tril()
    junk[low] = torch.randn(N, N, device=cuda_dev, generator=g)[low] * 1e30       # lower triangle and diagonal
    big = torch.full((N, N + 37), float("nan"), device=cuda_dev)
    big[:, :N] = Sd
    strided = big[:, :N]
    assert strided.stride(0) == N + 37
    # interleaved scoring calls, on the same handle's other plans
    E = torch.randn(600, 128, device=cuda_dev, generator=g)
    G = torch.randn(3000, 128, device=cuda_dev, generator=g)
    cs_ref, tk_ref = EN.cohort_stats(E, G, 50), EN.cosine_topk(E, G, 10)
    for m, (Z, lab) in ref.items():
        for X in (junk, strided):
            Z2, lab2 = EN.ahc(X, m, num_clusters=5)
            assert np.array_equal(Z, Z2) and torch.equal(lab, lab2), m
        cs = EN.cohort_stats(E, G, 50)
        Z2, lab2 = EN.ahc(Sd, m, num_clusters=5)
        tk = EN.cosine_topk(E, G, 10)
        assert np.array_equal(Z, Z2) and torch.equal(lab, lab2), m
        assert all(torch.equal(a, b) for a, b in zip(cs, cs_ref)) and all(torch.equal(a, b) for a, b in zip(tk, tk_ref))


def test_non_finite_similarity_raises(cuda_dev):
    S = torch.from_numpy(_sims(300, 4, "random")).to(cuda_dev)
    for bad in (float("nan"), float("inf"), float("-inf")):
        X = S.clone()
        X[17, 250] = bad
        with pytest.raises(RuntimeError, match="non-finite"):
            EN.ahc(X)
    X = S.clone()
    X[250, 17] = float("nan")                     # lower triangle: not read
    X[5, 5] = float("inf")
    Z, _ = EN.ahc(X)
    assert np.array_equal(Z, EN.ahc(S)[0])


# ---- diarize ----------------------------------------------------------------------------------------------------------
def _model():
    sd = RO.make_state_dict(0, num_classes=16)
    m = dsk.DeepSpeakerModel(512, 16).cuda()
    m.load_state_dict(sd)
    return m.eval()


def test_window_embeddings_match_the_forward(cuda_dev):
    g = np.random.RandomState(2)
    bank = F.FeatureBank.from_arrays([g.randn(n, 64) for n in (100, 700, 1234, 161)])
    model = _model()
    utt = np.array([2, 0, 3, 1])
    for batch in (7, 256):
        emb, wu, ws, wo = F.window_embeddings(model, bank, utt, T=160, hop=40, batch=batch)
        wu2, ws2, wo2 = bank.windows(utt, 160, 40)
        assert torch.equal(wu, wu2) and torch.equal(ws, ws2) and torch.equal(wo, wo2)
        W = wu.numel()
        Bb = min(batch, W)
        nb = -(-W // Bb)
        pad = nb * Bb - W
        wu_p, ws_p = torch.cat([wu, wu[-1:].expand(pad)]), torch.cat([ws, ws[-1:].expand(pad)])
        with torch.no_grad():
            ref = torch.cat([model(bank.crops(wu_p[i * Bb:(i + 1) * Bb], ws_p[i * Bb:(i + 1) * Bb], 160))
                             for i in range(nb)])[:W]
        assert torch.equal(emb, ref), batch


def _host_diarize(model, bank, utt, T, hop, k=None, t=None, method="average"):
    emb, _, ws, wo = F.window_embeddings(model, bank, utt, T, hop)
    out = []
    for r, u in enumerate(utt):
        a, b = int(wo[r]), int(wo[r + 1])
        if b - a == 1:
            wl = np.zeros(1, np.int32)
        else:
            E = emb[a:b]
            Zs = _scipy(EN.cosine_matrix(E, E).cpu().numpy(), method)
            wl = _relabel(fcluster(Zs, min(k, b - a), "maxclust") if k is not None else fcluster(Zs, t, "distance"))
        fl = O.frame_labels_brute(ws[a:b].numpy(), wl, int(bank.lengths[u]), T)
        out.append((fl, O.segments_brute(fl)))
    return out


def test_diarize_matches_a_host_recomposition(cuda_dev):
    g = np.random.RandomState(8)
    lens = [3000, 100, 1777, 161, 2400]
    bank = F.FeatureBank.from_arrays([g.randn(n, 64) for n in lens])
    model = _model()
    utt = [4, 0, 1, 2, 3]
    # a threshold that leaves 6 clusters in the first recording (the others fall where they fall)
    emb, _, _, wo = F.window_embeddings(model, bank, utt[:1], 160, 40)
    Zf, _ = EN.ahc(EN.cosine_matrix(emb, emb))
    t = float(Zf[-6:-4, 2].mean())
    for kw in ({"k": 3}, {"t": t}):
        got = DZ.diarize(model, bank, utt, T=160, hop=40, num_speakers=kw.get("k"), threshold=kw.get("t"))
        ref = _host_diarize(model, bank, utt, 160, 40, **kw)
        for r, (res, (fl, segs)) in enumerate(zip(got, ref)):
            assert np.array_equal(res.frame_labels, fl), (kw, r)
            assert res.segments == segs, (kw, r)
        print(f"\n{kw}: speakers per recording {[int(x.window_labels.max()) + 1 for x in got]}")
    per = DZ.diarize(model, bank, utt, num_speakers=[2, 1, 4, 3, 2])
    # frames 2400, 3000, 100 (one window: one speaker), 1777, 161 (two windows)
    assert [int(x.window_labels.max()) + 1 for x in per] == [2, 1, 1, 3, 2]
    with pytest.raises(ValueError, match="hop"):
        DZ.diarize(model, F.FeatureBank.from_arrays([np.zeros((40000, 64))]), [0], hop=1, num_speakers=2)
    with pytest.raises(RuntimeError):
        DZ.diarize(model.train(), bank, utt, num_speakers=2)


def test_synthetic_timeline_frame_error_matches_fp64(cuda_dev):
    """K speakers take turns over a one-recording timeline; each window gets its majority speaker's centre plus noise.
    The GPU pipeline (cosine_matrix -> ahc -> frame labels) and the fp64 one (numpy cosines -> scipy) must score the
    same frame error after the optimal speaker mapping."""
    rng = np.random.default_rng(4)
    K, D, T, hop = 5, 512, 160, 40
    turns = rng.integers(300, 2000, 60)
    spk = np.concatenate([np.full(n, i % K if i < K else rng.integers(0, K)) for i, n in enumerate(turns)])
    n = spk.size
    _, ws, _ = F.sliding_windows([n], [0], T, hop)
    ws = ws.numpy()
    wspk = np.array([np.bincount(spk[s:s + T], minlength=K).argmax() for s in ws])
    C = rng.standard_normal((K, D))
    X = (C[wspk] + 0.9 * rng.standard_normal((ws.size, D))).astype(np.float32)
    Xd = torch.from_numpy(X).to(cuda_dev)
    Z, lab = EN.ahc(EN.cosine_matrix(Xd, Xd), "average", num_clusters=K)
    fl_gpu = DZ.frame_labels(ws, lab.cpu().numpy(), n, T)
    Xn = X.astype(np.float64)
    Xn /= np.linalg.norm(Xn, axis=1, keepdims=True)
    Zs = scipy_linkage(squareform(1.0 - Xn @ Xn.T, checks=False), "average")
    gap = Zs[ws.size - K, 2] - Zs[ws.size - K - 1, 2]       # the fp64 cut's margin
    fl_ref = DZ.frame_labels(ws, _relabel(fcluster(Zs, K, "maxclust")), n, T)

    def frame_error(fl):
        cm = np.zeros((K, fl.max() + 1))
        np.add.at(cm, (spk, fl), 1)
        r, c = linear_sum_assignment(-cm)
        return 1.0 - cm[r, c].sum() / n

    e_gpu, e_ref = frame_error(fl_gpu), frame_error(fl_ref)
    print(f"\nsynthetic timeline: {ws.size} windows, frame error GPU {e_gpu:.4f}, fp64 {e_ref:.4f}, cut margin {gap:.3e}")
    if gap > 4e-6:
        assert e_gpu == e_ref
        assert np.array_equal(fl_gpu, fl_ref)
