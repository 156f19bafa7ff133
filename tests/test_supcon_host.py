"""The supervised-contrastive loss without a GPU: the fp64 oracle's explicit gradient against torch autograd of the
textbook formula and against finite differences, NT-Xent as its two-views case, its invariances, the host-side valid
count and argument rejection."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import steps
from deepspeaker_pytorch_b200.model import SupConLoss, supcon_valid_count
from oracle import supcon_oracle as S


def _case(counts, D, seed, norm=10.0):
    """Rows of len(counts) labels with counts[k] rows each (a shared direction per label plus noise), shuffled, labels
    drawn from a wide int64 range."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randperm(10 ** 6, generator=g)[:len(counts)] * 1000 - 10 ** 8
    labels = torch.cat([torch.full((c,), int(i), dtype=torch.int64) for c, i in zip(counts, ids)])
    perm = torch.randperm(labels.numel(), generator=g)
    col = torch.cat([torch.full((c,), k) for k, c in enumerate(counts)])[perm]
    labels = labels[perm]
    E = torch.randn(labels.numel(), D, generator=g, dtype=torch.float64)
    E = norm * E / E.norm(dim=1, keepdim=True) + 6.0 * torch.randn(len(counts), D, generator=g, dtype=torch.float64)[col]
    return E, labels


def _autograd(E, labels, tau):
    Ed = E.clone().requires_grad_(True)
    loss = S.loss_autograd(Ed, labels, tau)
    loss.backward()
    return loss.detach(), Ed.grad


RAGGED = [1, 2, 3, 5, 17, 1, 4, 9, 2, 6, 1]      # groups of 1 to 17 rows, three singletons


@pytest.mark.parametrize("tau", [0.05, 0.1, 1.0, 10.0])
@pytest.mark.parametrize("kind", ["ragged", "one_label", "zero_row"])
def test_oracle_gradient_equals_autograd(kind, tau):
    if kind == "one_label":
        E, labels = _case([24], 64, seed=2)
    else:
        E, labels = _case(RAGGED, 64, seed=11)
    if kind == "zero_row":
        E[3] = 0.0
    loss, gE_ref = _autograd(E, labels, tau)
    oloss, _, _, _ = S.forward(E, labels, tau)
    gE = S.backward(E, labels, tau)
    assert abs(float(oloss - loss)) <= 1e-10 * max(1.0, abs(float(loss)))
    assert float((gE - gE_ref).norm() / gE_ref.norm()) <= 1e-10
    if kind != "zero_row":     # the zero row's gradient is divided by the 1e-12 floor; compare the others per row
        rel = (gE - gE_ref).norm(dim=1) / gE_ref.norm(dim=1).clamp_min(1e-300)
        assert float(rel.max()) <= 1e-9


@pytest.mark.parametrize("tau", [0.1, 1.0])
def test_oracle_gradient_agrees_with_finite_differences(tau):
    E, labels = _case([3, 1, 4, 2], 64, seed=5)
    gE = S.backward(E, labels, tau)
    f = lambda E_: float(S.forward(E_, labels, tau)[0])  # noqa: E731
    h = 1e-6
    rng = np.random.default_rng(0)
    for _ in range(12):
        i, d = int(rng.integers(E.shape[0])), int(rng.integers(E.shape[1]))
        Ep, Em = E.clone(), E.clone()
        Ep[i, d] += h
        Em[i, d] -= h
        fd = (f(Ep) - f(Em)) / (2 * h)
        assert abs(fd - float(gE[i, d])) <= 1e-6 * max(1.0, abs(fd)), (i, d, fd, float(gE[i, d]))


@pytest.mark.parametrize("tau", [0.05, 0.5])
def test_two_views_per_label_is_nt_xent(tau):
    """Every label exactly twice: the loss is NT-Xent, cross-entropy over the (N, N - 1) logits without the diagonal
    with the partner as the target."""
    B, D = 40, 64
    g = torch.Generator().manual_seed(4)
    base = torch.randn(B, D, generator=g, dtype=torch.float64)
    E = torch.cat([base + 0.3 * torch.randn(B, D, generator=g, dtype=torch.float64),
                   base + 0.3 * torch.randn(B, D, generator=g, dtype=torch.float64)])
    labels = torch.arange(B).repeat(2)
    N = 2 * B
    z = F.normalize(E)
    logits = (z @ z.T) / tau
    off = ~torch.eye(N, dtype=torch.bool)
    logits = logits[off].reshape(N, N - 1)
    partner = (torch.arange(N) + B) % N
    target = partner - (partner > torch.arange(N)).long()     # the column index once the diagonal is gone
    ref = F.cross_entropy(logits, target)
    loss, _, _, _ = S.forward(E, labels, tau)
    assert abs(float(loss - ref)) <= 1e-12 * max(1.0, abs(float(ref)))


def test_relabel_and_permute():
    E, labels = _case([3, 2, 5, 1, 4], 64, seed=8)
    tau = 0.2
    loss, _, lse, rows = S.forward(E, labels, tau)
    gE = S.backward(E, labels, tau)
    relabel = {int(v): 7 - 13 * k for k, v in enumerate(torch.unique(labels).flip(0))}
    lab2 = torch.tensor([relabel[int(v)] for v in labels])
    loss2, _, lse2, rows2 = S.forward(E, lab2, tau)
    assert torch.equal(loss, loss2) and torch.equal(lse, lse2) and torch.equal(rows, rows2)
    assert torch.equal(S.backward(E, lab2, tau), gE)
    perm = torch.randperm(E.shape[0], generator=torch.Generator().manual_seed(1))
    loss3, _, lse3, rows3 = S.forward(E[perm], labels[perm], tau)
    gE3 = S.backward(E[perm], labels[perm], tau)
    assert abs(float(loss - loss3)) <= 1e-12
    assert float((lse3 - lse[perm]).abs().max()) <= 1e-12 and float((rows3 - rows[perm]).abs().max()) <= 1e-12
    assert float((gE3 - gE[perm]).abs().max()) <= 1e-12 * float(gE.abs().max())


def test_valid_count_matches_brute_force():
    rng = np.random.default_rng(3)
    for _ in range(50):
        n = int(rng.integers(1, 40))
        labels = rng.integers(-3, 6, n) * (2 ** 40)
        brute = sum(1 for i in range(n) if any(labels[j] == labels[i] for j in range(n) if j != i))
        assert supcon_valid_count(torch.from_numpy(labels)) == brute == S.valid_count(labels)
    assert supcon_valid_count([5, 5, 5]) == 3                      # one label: every row is valid
    assert supcon_valid_count([1, 2, 3]) == 0
    with pytest.raises(ValueError):
        supcon_valid_count(torch.tensor([0.5, 0.5]))


def test_bad_arguments_raise_before_any_device_work():
    """The embeddings are not even on a GPU: every check runs on the host first."""
    E = torch.empty(4, 64, device="meta")
    for t in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            SupConLoss(t)
    crit = SupConLoss(0.1)
    with pytest.raises(ValueError):                        # V = 0
        crit.forward(E, torch.tensor([1, 2, 3, 4]))
    with pytest.raises(RuntimeError):                      # label count
        crit.forward(E, torch.tensor([1, 1, 2]))
    with pytest.raises(RuntimeError):                      # a valid batch reaches the device check
        crit.forward(E, torch.tensor([1, 1, 2, 2]))

    class _Model:
        training = True

        def __call__(self, x):
            raise AssertionError("the step must reject the batch before the forward")

    with pytest.raises(ValueError):
        steps.supcon_step(_Model(), None, E, torch.tensor([1, 2, 3, 4]), temperature=0.1)
    with pytest.raises(ValueError):
        steps.supcon_step(_Model(), None, E, torch.tensor([1, 1, 2, 2]), temperature=math.inf)


def test_c_abi_rejects_bad_arguments_without_a_launch():
    lib = L.load()
    good = dict(N=8, D=64, V=8, tau=0.1)
    for bad in ({"N": 1}, {"N": L.DSK_SUPCON_MAX_N + 1}, {"D": 96}, {"V": 0}, {"V": 9}, {"tau": 0.0}, {"tau": -1.0},
                {"tau": float("nan")}, {"tau": float("inf")}):
        a = {**good, **bad}
        assert lib.dsk_supcon(None, 1, 1, a["N"], a["D"], a["V"], a["tau"], 1, 1, 1, None) == L.DSK_ERR_INVALID
        assert b"dsk_supcon" in lib.dsk_last_error()
        assert lib.dsk_supcon_bwd(None, 1, 1, 1, 1, a["N"], a["D"], a["V"], a["tau"], 1, 1, None) == L.DSK_ERR_INVALID
        assert b"dsk_supcon_bwd" in lib.dsk_last_error()
    assert lib.dsk_supcon(None, None, 1, 8, 64, 8, 0.1, 1, 1, 1, None) == L.DSK_ERR_INVALID    # null pointer
    assert lib.dsk_supcon(None, 1, 1, 8, 64, 8, 0.1, 1, 1, 1, None) == L.DSK_ERR_INVALID       # null handle
