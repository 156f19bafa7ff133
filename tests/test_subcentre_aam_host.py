"""Sub-centre AAM-softmax with the inter-top-k penalty without a GPU: the fp64 oracle against the plain AAM oracle at
K = 1, topk = 0 and against torch autograd of the textbook form, the tie and NaN rules of the sub-centre max and the
top-k selection, psi at cos = +-1, and argument rejection in the Python layer and the C ABI."""
import ctypes
import math

import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import engine as EN
from oracle import aam_softmax_oracle as A
from oracle import subcentre_aam_oracle as S


def _case(N, C, K, D, seed):
    g = torch.Generator().manual_seed(seed)
    E = torch.randn(N, D, generator=g, dtype=torch.float64)
    E = 10.0 * E / E.norm(dim=1, keepdim=True)
    W = torch.randn(C * K, D, generator=g, dtype=torch.float64) * 0.05
    return E, W, torch.randint(0, C, (N,), generator=g)


def test_k1_topk0_is_the_aam_oracle_bit_for_bit():
    E, W, y = _case(40, 23, 1, 64, seed=1)
    for m, s in ((0.0, 30.0), (0.2, 30.0), (0.5, 64.0)):
        loss, cos, lse, sub, top = S.forward(E, W, y, 1, m, s)
        aloss, acos, alse = A.forward(E, W, y, m, s)
        assert torch.equal(loss, aloss) and torch.equal(cos, acos) and torch.equal(lse, alse)
        assert not bool(sub.any()) and top.shape == (40, 0)
        gE, gW = S.backward(E, W, y, 1, m, s, grad_loss=0.7)
        aE, aW = A.backward(E, W, y, m, s, grad_loss=0.7)
        assert torch.equal(gE, aE) and torch.equal(gW, aW)


@pytest.mark.parametrize("K", [1, 2, 3, 5])
def test_explicit_backward_equals_autograd(K):
    C = 13
    for topk in (0, 1, 5):
        for tm in (0.0, 0.1):
            for m in (0.0, 0.2, 0.5):
                E, W, y = _case(32, C, K, 64, seed=1000 * K + 100 * topk + int(10 * tm) + int(100 * m))
                if m > 0:                                   # rows past pi - m: near their negated target sub-centres
                    gn = torch.Generator().manual_seed(3)
                    for k in range(1, K):
                        W[y[:4] * K + k] = W[y[:4] * K] + 0.005 * torch.randn(4, 64, dtype=torch.float64, generator=gn)
                    wy = W[y[:4] * K] / W[y[:4] * K].norm(dim=1, keepdim=True)
                    E[:4] = -10.0 * wy + 0.1 * torch.randn(4, 64, dtype=torch.float64, generator=gn)
                Ed, Wd = E.clone().requires_grad_(True), W.clone().requires_grad_(True)
                ref = S.loss_autograd(Ed, Wd, y, K, m, 30.0, topk, tm)
                ref.backward()
                ref = ref.detach()
                loss, cos, _, _, top = S.forward(E, W, y, K, m, 30.0, topk, tm)
                gE, gW = S.backward(E, W, y, K, m, 30.0, topk, tm)
                what = (K, topk, tm, m)
                assert abs(float(loss - ref)) <= 1e-10 * max(1.0, float(ref)), what
                assert float((gE - Ed.grad).abs().max()) <= 1e-10 * float(Ed.grad.abs().max()), what
                assert float((gW - Wd.grad).abs().max()) <= 1e-10 * float(Wd.grad.abs().max()), what
                if m > 0:
                    assert bool((cos[torch.arange(4), y[:4]] < A._consts(m)[2]).all()), what


def test_unchosen_subcentres_get_zero_weight_gradient():
    K, C = 3, 7
    E, W, y = _case(5, C, K, 64, seed=4)
    _, _, _, sub, _ = S.forward(E, W, y, K, 0.2, 30.0, 2, 0.1)
    _, gW = S.backward(E, W, y, K, 0.2, 30.0, 2, 0.1)
    chosen = torch.zeros(C * K, dtype=torch.bool)
    chosen[(torch.arange(C)[None, :] * K + sub).reshape(-1)] = True
    assert not bool(gW[~chosen].any()) and bool(gW[chosen].abs().sum(1).gt(0).all())


def test_subcentre_max_ties_and_nan():
    nan = math.nan
    g = torch.tensor([[0.5, 0.5, 0.3,   0.2, nan, 0.9,   nan, 0.9, nan,   0.1, 0.4, 0.4]], dtype=torch.float64)
    cos, sub = S.subcentre_max(g, 3)
    assert sub.tolist() == [[0, 1, 0, 1]]
    assert cos[0, 0] == 0.5 and math.isnan(cos[0, 1]) and math.isnan(cos[0, 2]) and cos[0, 3] == 0.4
    # duplicate sub-centre rows: the lower k wins
    E, W, y = _case(6, 4, 3, 64, seed=2)
    W[2::3] = W[0::3]
    _, cos, _, sub, _ = S.forward(E, W, y, 3, 0.2, 30.0)
    assert not bool((sub == 2).any())


def test_selection_ties_nan_and_target():
    nan = math.nan
    cos = torch.tensor([[0.3, 0.7, 0.3, nan, 0.7, -0.0, 0.0, 0.9, nan],
                        [nan, nan, 0.1, nan, nan, nan, nan, -math.inf, nan]], dtype=torch.float64)
    y = torch.tensor([7, 2])
    assert S.select_topk(cos, y, 8)[0].tolist() == [1, 4, 0, 2, 5, 6, 3, 8]   # ties to the lower c, -0 == +0, NaN last
    assert S.select_topk(cos, y, 3)[1].tolist() == [7, 0, 1]                    # -inf before NaN; target never chosen


def test_psi_at_the_poles():
    for tm in (0.0, 0.1, 0.4):
        c = torch.tensor([1.0, -1.0], dtype=torch.float64)
        assert S.psi(c, tm).tolist() == [math.cos(tm), -math.cos(tm)]
        assert S.dpsi(c, tm).tolist() == [math.cos(tm), math.cos(tm)]
    # a non-target class in T_i exactly on the row (cos = 1): the explicit gradient is finite
    E, W, y = _case(4, 6, 2, 64, seed=9)
    u = torch.zeros(64, dtype=torch.float64)
    u[3] = 1.0
    y[0] = 0
    E[0], W[2 * 4 + 1] = 10.0 * u, 0.25 * u
    _, cos, _, sub, top = S.forward(E, W, y, 2, 0.2, 30.0, 2, 0.1)
    assert cos[0, 4] == 1.0 and sub[0, 4] == 1 and top[0, 0] == 4
    gE, gW = S.backward(E, W, y, 2, 0.2, 30.0, 2, 0.1)
    assert bool(torch.isfinite(gE).all()) and bool(torch.isfinite(gW).all())


def test_python_layer_rejects_bad_arguments():
    W = torch.zeros(30, 64)
    good = dsk.AAMSoftmaxLoss(W, 0.2, 30.0, subcentres=3, topk=9, topk_margin=0.1)
    assert (good.subcentres, good.topk, good.topk_margin) == (3, 9, 0.1)
    dsk.AAMSoftmaxLoss(W, 0.2, 30.0)
    bad = [dict(subcentres=0), dict(subcentres=17), dict(subcentres=4), dict(subcentres=2.0), dict(subcentres=True),
           dict(subcentres=3, topk=10), dict(topk=65), dict(topk=-1), dict(topk=1.5), dict(topk_margin=-0.1),
           dict(topk_margin=math.nan), dict(topk_margin=math.inf)]
    for kw in bad:
        with pytest.raises(ValueError):
            dsk.AAMSoftmaxLoss(torch.zeros(30 if kw.get("topk") != 65 else 100, 64), 0.2, 30.0, **kw)
    with pytest.raises(ValueError):
        EN.subcentre_cosines(torch.zeros(4, 64), torch.zeros(10, 64), torch.zeros(4, dtype=torch.long), 3)


P = ctypes.c_void_p(256)                                 # never dereferenced: the arguments are checked first


def _rejected(rc, what):
    assert rc == -1, (what, rc)
    assert b"bad arguments" in L.load().dsk_last_error(), what


def test_c_abi_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    # dsk_aam_softmax_sc(h, E, W, labels, N, C, K, D, m, s, topk, m', loss, cos, lse, sub, top, stream)
    ok = dict(N=8, C=100, K=3, D=64, m=0.2, s=30.0, topk=5, tm=0.1, sub=P, top=P)
    cases = {"K = 0": dict(K=0), "K = 17": dict(K=17), "C K > 65536": dict(C=21846), "C = 1": dict(C=1, topk=0),
             "topk = C": dict(C=5, topk=5), "topk = 65": dict(topk=65), "topk < 0": dict(topk=-1),
             "m' < 0": dict(tm=-0.1), "m' nan": dict(tm=math.nan), "m' inf": dict(tm=math.inf),
             "null sub at K = 3": dict(sub=None), "null top at topk = 5": dict(top=None), "D % 64": dict(D=96)}
    for what, kw in cases.items():
        a = {**ok, **kw}
        _rejected(lib.dsk_aam_softmax_sc(P, P, P, P, a["N"], a["C"], a["K"], a["D"], a["m"], a["s"], a["topk"], a["tm"],
                                         P, P, P, a["sub"], a["top"], None), "fwd " + what)
        _rejected(lib.dsk_aam_softmax_sc_bwd(P, P, P, P, P, P, a["sub"], a["top"], a["N"], a["C"], a["K"], a["D"],
                                             a["m"], a["s"], a["topk"], a["tm"], P, P, P, None), "bwd " + what)
    # dsk_aam_subcentre_cos(E, W, labels, N, C, K, D, out, stream)
    for what, a in {"null E": (None, P, P, 4, 10, 3, 64, P), "null out": (P, P, P, 4, 10, 3, 64, None),
                    "N = 0": (P, P, P, 0, 10, 3, 64, P), "K = 0": (P, P, P, 4, 10, 0, 64, P),
                    "K = 17": (P, P, P, 4, 10, 17, 64, P), "D = 0": (P, P, P, 4, 10, 3, 0, P)}.items():
        _rejected(lib.dsk_aam_subcentre_cos(*a, None), "subcentre_cos " + what)
