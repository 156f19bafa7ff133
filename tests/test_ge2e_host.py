"""GE2E without a GPU: the fp64 oracle's explicit gradients against torch autograd of the textbook formula and against
finite differences, its invariances, and the host-side speaker lists the loss builds from the labels."""
import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200.model import GE2ELoss, ge2e_batch
from oracle import ge2e_oracle as G


def _case(counts, D, seed, norm=10.0):
    """Rows of len(counts) speakers with counts[k] rows each, shuffled, labels drawn from a wide int64 range."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randperm(10 ** 6, generator=g)[:len(counts)] * 1000 - 10 ** 8
    labels = torch.cat([torch.full((c,), int(i), dtype=torch.int64) for c, i in zip(counts, ids)])
    labels = labels[torch.randperm(labels.numel(), generator=g)]
    E = torch.randn(labels.numel(), D, generator=g, dtype=torch.float64)
    E = norm * E / E.norm(dim=1, keepdim=True)
    # speaker structure: rows of one speaker share a direction
    centre = torch.randn(len(counts), D, generator=g, dtype=torch.float64)
    col, _, _ = G.speakers(labels)
    E = E + 2.0 * centre[col]
    return E, labels


def _autograd(E, labels, w, b, method):
    Ed = E.clone().requires_grad_(True)
    wd = torch.tensor(float(w), dtype=torch.float64, requires_grad=True)
    bd = torch.tensor(float(b), dtype=torch.float64, requires_grad=True)
    loss = G.loss_autograd(Ed, labels, wd, bd, method)
    loss.backward()
    return loss.detach(), Ed.grad, float(wd.grad), float(bd.grad)


COUNTS = [1, 2, 3, 5, 17, 1, 4, 9, 2, 6]     # unequal n_k from 1 to 17, two singleton speakers


@pytest.mark.parametrize("method", ["softmax", "contrast"])
@pytest.mark.parametrize("w,b", [(10.0, -5.0), (0.5, 3.0), (1e-7, -5.0)], ids=["w10", "w0.5", "w_clamped"])
def test_oracle_gradients_equal_autograd(method, w, b):
    E, labels = _case(COUNTS, 64, seed=11)
    loss, gE_ref, gw_ref, gb_ref = _autograd(E, labels, w, b, method)
    oloss, _, _ = G.forward(E, labels, w, b, method)
    gE, gw, gb = G.backward(E, labels, w, b, method)
    assert abs(float(oloss - loss)) <= 1e-10 * max(1.0, abs(float(loss)))
    assert float((gE - gE_ref).norm() / gE_ref.norm()) <= 1e-10
    if w < 1e-6:
        assert gw == 0.0 and gw_ref == 0.0
    else:
        assert abs(gw - gw_ref) <= 1e-10 * max(abs(gw_ref), 1e-6)
    if method == "softmax":
        assert gb == 0.0                                   # exactly; autograd leaves a rounding residue
        assert abs(gb_ref) <= 1e-12
    else:
        assert abs(gb - gb_ref) <= 1e-10 * max(abs(gb_ref), 1e-6)    # a sum of cancelling terms


@pytest.mark.parametrize("method", ["softmax", "contrast"])
def test_oracle_gradients_agree_with_finite_differences(method):
    E, labels = _case([3, 1, 4, 2], 64, seed=5)
    w, b = 2.0, -1.0
    gE, gw, gb = G.backward(E, labels, w, b, method)
    f = lambda E_, w_=w, b_=b: float(G.forward(E_, labels, w_, b_, method)[0])  # noqa: E731
    h = 1e-6
    rng = np.random.default_rng(0)
    for _ in range(12):
        i, d = int(rng.integers(E.shape[0])), int(rng.integers(E.shape[1]))
        Ep, Em = E.clone(), E.clone()
        Ep[i, d] += h
        Em[i, d] -= h
        fd = (f(Ep) - f(Em)) / (2 * h)
        assert abs(fd - float(gE[i, d])) <= 1e-6 * max(1.0, abs(fd)), (i, d, fd, float(gE[i, d]))
    assert abs((f(E, w + h) - f(E, w - h)) / (2 * h) - gw) <= 1e-6
    if method == "contrast":
        assert abs((f(E, w, b + h) - f(E, w, b - h)) / (2 * h) - gb) <= 1e-6


def test_exclusive_centroid_of_a_pair_is_the_other_row():
    E, labels = _case([2, 2, 3], 64, seed=3)
    e, _, _, cx, col, n, valid = G.centroids(E, labels)
    for i in range(E.shape[0]):
        if n[col[i]] == 2:
            j = [u for u in range(E.shape[0]) if col[u] == col[i] and u != i][0]
            assert torch.equal(cx[i], e[j])


@pytest.mark.parametrize("method", ["softmax", "contrast"])
def test_relabel_and_permute(method):
    E, labels = _case([3, 2, 5, 1, 4], 64, seed=8)
    loss, _, _ = G.forward(E, labels, 3.0, -2.0, method)
    gE, gw, gb = G.backward(E, labels, 3.0, -2.0, method)
    perm = torch.randperm(E.shape[0], generator=torch.Generator().manual_seed(1))
    relabel = {int(v): 7 - 13 * k for k, v in enumerate(torch.unique(labels).flip(0))}   # reverses the speaker order
    lab2 = torch.tensor([relabel[int(v)] for v in labels[perm]])
    loss2, _, _ = G.forward(E[perm], lab2, 3.0, -2.0, method)
    gE2, gw2, gb2 = G.backward(E[perm], lab2, 3.0, -2.0, method)
    assert abs(float(loss - loss2)) <= 1e-12
    assert float((gE2 - gE[perm]).abs().max()) <= 1e-12 * float(gE.abs().max())
    assert abs(gw - gw2) <= 1e-12 * max(abs(gw), 1.0) and abs(gb - gb2) <= 1e-12 * max(abs(gb), 1.0)


def test_host_speaker_lists_from_arbitrary_labels():
    labels = torch.tensor([2 ** 40, -7, 5, -7, 2 ** 40, 0, 5, 5, -(2 ** 50)], dtype=torch.int64)
    order, offsets, col, V = ge2e_batch(labels)
    ids = np.unique(labels.numpy())
    assert offsets.tolist() == [0, 1, 3, 4, 7, 9]
    for k in range(ids.size):
        rows = order[offsets[k]:offsets[k + 1]]
        assert (labels.numpy()[rows] == ids[k]).all() and (np.diff(rows) > 0).all()
        assert (col[rows] == k).all()
    assert V == 7                                          # -2^50 and 0 are singletons
    o2, off2, col2 = G.host_csr(labels)
    assert (o2 == order).all() and (off2 == offsets).all() and (col2 == col).all()
    assert ge2e_batch(np.array([3, 3, 3]))[3] == 0         # one speaker
    assert ge2e_batch([1, 2, 3])[3] == 0                   # no speaker with two rows
    with pytest.raises(ValueError):
        ge2e_batch(torch.tensor([0.5, 1.5]))


def test_no_valid_row_raises_before_any_device_work():
    """V = 0 (P < 2, or only singletons) raises ValueError from the labels alone, before the embeddings are looked at
    (these are not even on a GPU)."""
    crit = GE2ELoss()
    E = torch.empty(4, 64, device="meta")
    for labels in ([1, 1, 1, 1], [1, 2, 3, 4]):
        with pytest.raises(ValueError):
            crit.forward(E, torch.tensor(labels))
    with pytest.raises(RuntimeError):                      # a valid batch reaches the device check
        crit.forward(E, torch.tensor([1, 1, 2, 2]))
    with pytest.raises(ValueError):
        GE2ELoss(method="angular")


def test_c_abi_rejects_bad_arguments_without_a_launch():
    lib = L.load()
    assert lib.dsk_ge2e(None, None, 8, 64, None, None, None, 2, 4, None, None, 0, None, None, None, None) < 0
    assert lib.dsk_ge2e_bwd(None, None, 8, 64, None, None, None, 2, 4, None, None, 0, None, None, None, None, None, None,
                            None) < 0
    assert b"dsk_ge2e" in lib.dsk_last_error()
