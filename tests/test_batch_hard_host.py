"""Batch-hard triplet loss, host side: the C oracle against an fp64 numpy restatement, its tie rule, the number of
valid anchors from the labels and the rejection of a batch without any."""
import types

import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200.model import batch_hard_valid_count
from deepspeaker_pytorch_b200.steps import batch_hard_step
from oracle import batch_hard_oracle as BH


def _numpy_fp64(E, labels, margin):
    E = E.astype(np.float64)
    N, D = E.shape
    d = np.sqrt(((E[:, None, :] - E[None, :, :]) ** 2).sum(-1) + 1e-4 / D)
    same = labels[:, None] == labels[None, :]
    pos = np.where(same & ~np.eye(N, dtype=bool), d, -np.inf).argmax(1)
    neg = np.where(~same, d, np.inf).argmin(1)
    valid = (same.sum(1) >= 2) & ((~same).sum(1) >= 1)
    h = np.maximum(margin + d[np.arange(N), pos] - d[np.arange(N), neg], 0.0)
    return h[valid].sum() / max(int(valid.sum()), 1), pos, neg, d, valid


@pytest.mark.parametrize("N,D,groups", [(96, 64, 8), (130, 96, 13), (40, 512, 4)])
def test_c_oracle_matches_fp64_on_separated_inputs(N, D, groups):
    rng = np.random.default_rng(N)
    labels = np.arange(N) % groups
    labels[-1] = groups + 5                                   # a singleton speaker: an invalid anchor
    # distinct pairwise distances (gaps far above fp32 rounding): the argmax/argmin are unambiguous
    E = (rng.standard_normal((N, D)) * np.linspace(1.0, 3.0, N)[:, None]).astype(np.float32)
    loss, pos, neg, d_ap, d_an, valid = BH.batch_hard_triplet(E, labels, 1.0)
    rloss, rpos, rneg, rd, rvalid = _numpy_fp64(E, labels, 1.0)
    assert np.array_equal(valid, rvalid) and not valid[-1] and valid.sum() == N - 1
    assert np.array_equal(pos[valid], rpos[valid]) and np.array_equal(neg, rneg)
    assert pos[-1] == -1 and d_ap[-1] == 0.0
    assert np.allclose(d_ap[valid], rd[np.arange(N), rpos][valid], rtol=1e-6)
    assert np.allclose(d_an, rd[np.arange(N), rneg], rtol=1e-6)
    assert abs(loss - rloss) <= 1e-5 * max(1.0, rloss)


def test_c_oracle_ties_go_to_the_lower_index_and_empty_batches():
    rng = np.random.default_rng(1)
    base = rng.standard_normal((6, 32)).astype(np.float32)
    E = np.concatenate([base, base])                          # row r and row r+6 are identical
    labels = np.array([0, 1, 2, 0, 1, 2, 3, 4, 5, 3, 4, 5])
    _, pos, neg, d_ap, d_an, valid = BH.batch_hard_triplet(E, labels, 0.5)
    assert valid.all()
    for i in range(12):
        same = [j for j in range(12) if labels[j] == labels[i] and j != i]
        other = [j for j in range(12) if labels[j] != labels[i]]
        dist = lambda j: float(np.sqrt(np.sum((E[i].astype(np.float64) - E[j]) ** 2) + 1e-4 / 32))
        assert pos[i] == min(same, key=lambda j: (-dist(j), j))
        assert neg[i] == min(other, key=lambda j: (dist(j), j))
    assert neg[0] == 6 and neg[6] == 0                         # exact duplicates of another label: distance sqrt(eps)
    E2 = np.stack([base[0], base[1], base[1], base[2], base[2]])
    _, pos, neg, _, _, _ = BH.batch_hard_triplet(E2, np.array([0, 0, 0, 1, 1]), 0.5)
    assert pos[0] == 1 and neg[0] == 3                         # exact ties on both sides: the lower index
    loss, pos, neg, _, d_an, valid = BH.batch_hard_triplet(E, np.zeros(12, np.int64), 0.5)
    assert loss == 0.0 and not valid.any() and (neg == -1).all() and np.isinf(d_an).all()


def test_valid_count_from_labels():
    assert batch_hard_valid_count(torch.arange(16) % 4) == 16
    assert batch_hard_valid_count(torch.tensor([0, 0, 1, 2, 3, 3, 3])) == 5     # singletons 1, 2 are not anchors
    assert batch_hard_valid_count(torch.tensor([7, 7, 7, 7])) == 0               # one speaker: no negatives
    assert batch_hard_valid_count(torch.arange(8)) == 0                          # no speaker twice: no positives
    assert batch_hard_valid_count([3, 3, 5]) == 2


@pytest.mark.parametrize("labels", [torch.arange(8), torch.zeros(8, dtype=torch.long)])
def test_step_rejects_a_batch_without_valid_anchors(labels):
    model = types.SimpleNamespace(training=True)                # rejected before any forward
    with pytest.raises(ValueError):
        batch_hard_step(model, None, None, labels, margin=0.5)
