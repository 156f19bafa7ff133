"""VBx and the frame-level DER on the host (no GPU): the oracle's full-matrix forward-backward against a brute-force sum
over all state paths and against a rank-one restatement of the recursion (the one the kernel runs), the ELBO's
monotonicity, dsk_vbx's argument checks, the Python entry points' errors, and ``der`` against brute force."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import diarization as DZ
from deepspeaker_pytorch_b200 import engine as EN
from oracle import vbx_oracle as O

P = ctypes.c_void_p(256)                                 # never dereferenced: the arguments are checked first
LOOPS = [0.0, 0.3, 0.9, 1.0]


def _case(rng, W, S):
    lnp = rng.normal(size=(W, S)) * 3.0
    pi = rng.dirichlet(np.ones(S))
    return lnp, pi


def _brute(lnp, pi, loop_p):
    """(gamma, ln p(X), switch) by enumerating every state path."""
    W, S = lnp.shape
    A = loop_p * np.eye(S) + (1.0 - loop_p) * pi[None, :]
    paths, probs, sw = [], [], []
    for z in itertools.product(range(S), repeat=W):
        p = pi[z[0]] * np.exp(lnp[0, z[0]])
        s = np.zeros(S)
        for t in range(1, W):
            p *= A[z[t - 1], z[t]] * np.exp(lnp[t, z[t]])
            if loop_p < 1.0:                               # the share of the transition that is a switch into z_t
                s[z[t]] += (1.0 - loop_p) * pi[z[t]] / A[z[t - 1], z[t]]
        paths.append(z)
        probs.append(p)
        sw.append(s)
    probs = np.array(probs)
    px = probs.sum()
    post = probs / px
    gamma = np.zeros((W, S))
    for z, q in zip(paths, post):
        gamma[np.arange(W), z] += q
    return gamma, np.log(px), (post[:, None] * np.array(sw)).sum(axis=0)


def _rank_one(lnp, pi, loop_p):
    """The kernel's recursion: scaled messages in the log domain with the rank-one transition sum."""
    W, S = lnp.shape
    with np.errstate(divide="ignore"):
        lpi, lst, lsw = np.log(pi), np.log(loop_p), np.log(1.0 - loop_p)
    la = np.empty((W, S))
    lC = np.empty(W)
    for t in range(W):
        x = lnp[t] + (lpi if t == 0 else np.logaddexp(lst + la[t - 1], lsw + lpi))
        m = x.max()
        c = np.exp(x - m).sum()
        la[t] = x - m - np.log(c)
        lC[t] = m + np.log(c)
    lb = np.zeros(S)
    gamma = np.empty((W, S))
    switch = np.zeros(S)
    for t in range(W - 1, -1, -1):
        gamma[t] = np.exp(la[t] + lb)
        if t == 0:
            break
        lu = lnp[t] + lb - lC[t]
        switch += np.exp(lsw + lpi + lu)
        v = lpi + lu
        M = v.max()
        lb = np.logaddexp(lst + lu, lsw + M + np.log(np.exp(v - M).sum()))
    return gamma, lC.sum(), switch


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(1.0, np.abs(np.asarray(b)).max())


@pytest.mark.parametrize("loop_p", LOOPS)
def test_full_matrix_forward_backward_equals_path_enumeration(loop_p):
    rng = np.random.default_rng(int(loop_p * 10))
    worst = 0.0
    for W in range(1, 8):
        for S in range(1, 4):
            lnp, pi = _case(rng, W, S)
            g, lpx, _, _, sw = O.forward_backward(lnp, pi, loop_p)
            gb, lpxb, swb = _brute(lnp, pi, loop_p)
            worst = max(worst, _rel(g, gb), abs(lpx - lpxb) / max(1.0, abs(lpxb)), _rel(sw, swb))
    print(f"loop_p {loop_p}: full matrix vs enumeration, max rel {worst:.2e}")
    assert worst < 1e-12


@pytest.mark.parametrize("loop_p", LOOPS)
def test_rank_one_recursion_equals_full_matrix(loop_p):
    rng = np.random.default_rng(100 + int(loop_p * 10))
    worst = 0.0
    for W, S in [(1, 1), (1, 4), (2, 3), (9, 5), (50, 17), (200, 64), (300, 128)]:
        lnp, pi = _case(rng, W, S)
        # unit emissions, then peaky ones: messages far outside fp64's linear range
        for scale in (1.0, 30.0):
            g, lpx, _, _, sw = O.forward_backward(scale * lnp, pi, loop_p)
            g1, lpx1, sw1 = _rank_one(scale * lnp, pi, loop_p)
            worst = max(worst, _rel(g1, g), abs(lpx1 - lpx) / max(1.0, abs(lpx)), _rel(sw1, sw))
    print(f"loop_p {loop_p}: rank one vs full matrix, max rel {worst:.2e}")
    assert worst < 1e-12


def _synthetic(rng, K, W, d, loop_p=0.99):
    """PLDA-space rows of an HMM over K speakers: x_t = sqrt(phi) o y_{z_t} + N(0, I), y_k ~ N(0, I)."""
    phi = np.sort(rng.gamma(2.0, 2.0, size=d))[::-1]
    Y = rng.normal(size=(K, d))
    z = np.empty(W, np.int64)
    z[0] = rng.integers(K)
    for t in range(1, W):
        z[t] = z[t - 1] if rng.random() < loop_p else rng.integers(K)
    return np.sqrt(phi) * Y[z] + rng.normal(size=(W, d)), phi, z


@pytest.mark.parametrize("seed", range(4))
def test_elbo_does_not_decrease(seed):
    rng = np.random.default_rng(seed)
    X, phi, z = _synthetic(rng, 2 + seed, 150, 12)
    init = (z * 3 + rng.integers(3, size=z.size)) % (3 * (2 + seed))   # an over-clustered start
    for loop_p in (0.0, 0.5, 0.99):
        r = O.vbx(X, phi, init, loop_p=loop_p, max_iters=15, epsilon=-np.inf)
        e = r["elbo"]
        drop = (e[:-1] - e[1:]) / np.abs(e[1:])
        print(f"seed {seed} loop_p {loop_p}: ELBO {e[0]:.3f} -> {e[-1]:.3f}, largest relative drop {drop.max():.2e}")
        assert r["iters"] == 15
        assert drop.max() <= 1e-9
        np.testing.assert_allclose(r["pi"].sum(), 1.0, rtol=1e-12)
        np.testing.assert_allclose(r["gamma"].sum(axis=1), 1.0, rtol=1e-10)


def test_oracle_stops_on_the_elbo_gain():
    rng = np.random.default_rng(9)
    X, phi, z = _synthetic(rng, 3, 200, 8)
    r = O.vbx(X, phi, z, max_iters=40, epsilon=1e-3)
    e = r["elbo"]
    assert r["iters"] == e.size
    assert np.all(np.diff(e)[:-1] >= 1e-3)
    assert r["iters"] == 40 or e[-1] - e[-2] < 1e-3


def _rejected(rc, what):
    assert rc == -1, (what, rc)
    assert b"bad arguments" in L.load().dsk_last_error(), what


def test_c_abi_rejects_bad_arguments_without_a_gpu():
    lib = L.load()

    def offs(*v):
        return (ctypes.c_int64 * len(v))(*v)

    good = dict(X=P, W=10, d=8, offsets=offs(0, 4, 10), R=2, labels=P, S=3, phi=P, Fa=0.3, Fb=17.0, loop_p=0.99,
                sm=5.0, max_iters=10, eps=1e-4, gamma=P, pi=P, elbo=P, iters=P, out=P)
    nan = float("nan")
    cases = {"null X": dict(X=None), "null offsets": dict(offsets=None), "null labels": dict(labels=None),
             "null phi": dict(phi=None), "null gamma": dict(gamma=None), "null pi": dict(pi=None),
             "null elbo": dict(elbo=None), "null iters": dict(iters=None), "null labels out": dict(out=None),
             "R = 0": dict(R=0, offsets=offs(0)), "d = 0": dict(d=0), "d > max": dict(d=L.DSK_F64_MAX_DIM + 1),
             "S = 0": dict(S=0), "S > max": dict(S=L.DSK_VBX_MAX_SPEAKERS + 1),
             "offsets[0] != 0": dict(offsets=offs(1, 4, 10)), "offsets[R] != W": dict(offsets=offs(0, 4, 9)),
             "empty recording": dict(offsets=offs(0, 4, 4, 10), R=3), "decreasing": dict(offsets=offs(0, 11, 10)),
             "recording too long": dict(W=L.DSK_AHC_MAX_N + 5, offsets=offs(0, 4, L.DSK_AHC_MAX_N + 5)),
             "Fa = 0": dict(Fa=0.0), "Fa < 0": dict(Fa=-1.0), "Fb = 0": dict(Fb=0.0), "loop_p < 0": dict(loop_p=-0.1),
             "loop_p > 1": dict(loop_p=1.5), "init_smoothing < 0": dict(sm=-1.0), "max_iters = 0": dict(max_iters=0),
             "NaN Fa": dict(Fa=nan), "NaN Fb": dict(Fb=nan), "NaN loop_p": dict(loop_p=nan),
             "NaN init_smoothing": dict(sm=nan), "NaN epsilon": dict(eps=nan)}
    for what, change in cases.items():
        a = dict(good, **change)
        _rejected(lib.dsk_vbx(a["X"], a["W"], a["d"], a["offsets"], a["R"], a["labels"], a["S"], a["phi"], a["Fa"],
                              a["Fb"], a["loop_p"], a["sm"], a["max_iters"], a["eps"], a["gamma"], a["pi"], a["elbo"],
                              a["iters"], a["out"], None), what)


def test_python_entry_points_reject_bad_arguments():
    with pytest.raises(RuntimeError):
        EN.vbx(torch.zeros(6, 4), [0, 6], np.zeros(6), np.ones(4), 0.3, 17.0, 0.99, 5.0, 10, 1e-4)   # CPU rows
    with pytest.raises(RuntimeError):
        DZ.vbx(None, torch.zeros(6, 4), [0, 6], np.zeros(6))                                        # CPU embeddings

    class _Eval:
        training = False

    with pytest.raises(ValueError, match="PLDA"):
        DZ.diarize(_Eval(), None, [0], num_speakers=2, vbx={})
    with pytest.raises(ValueError, match="unknown"):
        DZ.diarize(_Eval(), None, [0], num_speakers=2, plda=object(), vbx={"fa": 0.3})
    with pytest.raises(ValueError):
        DZ.diarize(_Eval(), None, [0], num_speakers=2, plda=object(), vbx=0.3)


def test_renumber_follows_first_appearance_per_recording():
    lab = np.array([4, 4, 1, 7, 1, 2, 2, 0, 5, -1, -1])
    np.testing.assert_array_equal(DZ._renumber(lab, [0, 5, 9, 11]), [0, 0, 1, 2, 1, 0, 0, 1, 2, -1, -1])


def _der_brute(ref, hyp):
    sp = ref >= 0
    n = sp.sum()
    miss = (sp & (hyp < 0)).sum()
    fa = (~sp & (hyp >= 0)).sum()
    both = sp & (hyp >= 0)
    R, H = sorted(set(ref[both])), sorted(set(hyp[both]))
    best = 0
    for choice in itertools.product(R + [None], repeat=len(H)):
        used = [c for c in choice if c is not None]
        if len(used) != len(set(used)):
            continue
        m = dict(zip(H, choice))
        best = max(best, sum(1 for r, h in zip(ref[both], hyp[both]) if m[h] == r))
    return (miss + fa + both.sum() - best) / n, miss / n, fa / n, (both.sum() - best) / n


def test_der_equals_brute_force_over_injective_mappings():
    rng = np.random.default_rng(5)
    for trial in range(60):
        n = int(rng.integers(1, 60))
        kr, kh = int(rng.integers(1, 6)), int(rng.integers(1, 6))
        ref = rng.integers(-1, kr, size=n)
        if not (ref >= 0).any():
            ref[0] = 0
        hyp = rng.integers(-1, kh, size=n)
        got = DZ.der(ref, hyp)
        want = _der_brute(ref, hyp)
        np.testing.assert_allclose((got.der, got.miss, got.false_alarm, got.confusion), want, rtol=0, atol=1e-15)
        assert len(set(got.mapping.values())) == len(got.mapping)


def test_der_hand_cases():
    ref = np.array([0, 0, 1, 1, 1, 2, -1, -1])
    r = DZ.der(ref, np.full(8, -1))                                      # all miss
    assert (r.der, r.miss, r.false_alarm, r.confusion, r.mapping) == (1.0, 1.0, 0.0, 0.0, {})
    r = DZ.der(np.array([0, 0, -1, -1, -1, -1]), np.array([0, 0, 3, 3, 3, 3]))   # every non-speech frame false alarm
    assert (r.der, r.miss, r.false_alarm, r.confusion) == (2.0, 0.0, 2.0, 0.0)
    perm = np.array([5, 9, 2])
    hyp = np.where(ref >= 0, perm[np.maximum(ref, 0)], -1)
    r = DZ.der(ref, hyp)                                                 # a perfect permutation
    assert r.der == 0.0 and r.mapping == {5: 0, 9: 1, 2: 2}
    with pytest.raises(ValueError, match="frames"):
        DZ.der(ref, hyp[:-1])
    with pytest.raises(ValueError, match="no speech"):
        DZ.der(np.full(4, -1), np.zeros(4))
