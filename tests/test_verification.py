"""Verification metric: restated sweep vs the reference's own eval_metrics (golden), and held-out EER parity of the
H100 engine vs the oracle on synthetic speakers (north star: EER within 0.1 % absolute)."""
import os

import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import verification as V
from oracle import rescnn_oracle as O
from oracle import verification_oracle as VO


def synthetic_pairs(P, crops, T, seed):
    """Same-speaker pairs share a base spectrogram (+ per-crop noise), different-speaker pairs do not."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(P, 1, T, 64, generator=g) * 4.0
    other = torch.randn(P, 1, T, 64, generator=g) * 4.0
    same = torch.arange(P) % 2 == 0
    a = base + 2.5 * torch.randn(P, crops, T, 64, generator=g)
    p = torch.where(same.view(P, 1, 1, 1), base, other) + 2.5 * torch.randn(P, crops, T, 64, generator=g)
    return a, p, same.numpy()


def test_sweep_matches_reference_eval_metrics(golden_dir):
    g = np.load(os.path.join(golden_dir, "verification.npz"))
    acc, eer = V.sweep(g["distances"], g["labels"])
    assert abs(acc - float(g["ref_accuracy"])) < 1e-12          # reference eval_metrics.evaluate (best-threshold accuracy)
    tpr, fpr, oacc = VO.evaluate_accuracy(g["distances"], g["labels"])
    assert abs(oacc - float(g["ref_accuracy"])) < 1e-12 and abs(tpr - float(g["ref_tpr"])) < 1e-12
    assert abs(eer - VO.equal_error_rate(g["distances"], g["labels"])) < 1e-12
    assert 0.0 < eer < 0.5


@pytest.mark.gpu
def test_heldout_eer_within_a_tenth_of_a_percent(cuda_dev):
    import deepspeaker_pytorch_b200 as dsk

    sd = O.make_state_dict(0, 16)
    m = dsk.DeepSpeakerModel(512, 16).to(cuda_dev).eval()
    m.load_state_dict(sd)
    P, crops, T = 96, 8, 32                       # 8 crops per file, 32-frame crops: the reference's own test setup
    a, p, same = synthetic_pairs(P, crops, T, seed=11)
    d_gpu = V.verification_distances(m, a.cuda(), p.cuda()).cpu().numpy()
    with torch.no_grad():
        ea = O.forward(sd, a.reshape(P * crops, 1, T, 64))
        ep = O.forward(sd, p.reshape(P * crops, 1, T, 64))
        d_ref = VO.crop_mean_distances(O.pairwise_distance(ea, ep).numpy(), P, crops)
    assert np.allclose(d_gpu, d_ref, rtol=2e-3, atol=2e-3)
    acc_g, eer_g = V.sweep(d_gpu, same)
    _, _, acc_r = VO.evaluate_accuracy(d_ref, same)
    eer_r = VO.equal_error_rate(d_ref, same)
    assert 0.0 <= eer_r < 0.5
    assert abs(eer_g - eer_r) <= 1e-3, (eer_g, eer_r)          # north star: within 0.1 % absolute
    assert abs(acc_g - acc_r) <= 1.0 / P + 1e-9


def test_oracle_val_at_far_matches_reference_ingredients(golden_dir):
    """VAL@FAR (eval_metrics.py:53-88): the oracle against the golden made from the reference's own calculate_val_far and
    scipy interp1d('slinear') on the de-duplicated FAR curve (the reference's calculate_val itself raises on duplicates)."""
    g = np.load(os.path.join(golden_dir, "verification.npz"))
    assert "duplicates" in str(g["ref_calculate_val_raises"])
    th = np.arange(0, 30, 0.001)
    for name, target in (("1e-2", 1e-2), ("5e-2", 5e-2)):
        val, far, thr = VO.calculate_val(th, g["distances"], g["labels"], target)
        assert abs(thr - float(g[f"val_threshold_{name}"])) < 1e-9
        assert val == float(g[f"val_{name}"]) and far == float(g[f"far_{name}"])


@pytest.mark.gpu
def test_gpu_evaluate_matches_reference_eval_metrics(cuda_dev, golden_dir):
    """verification.evaluate = eval_metrics.evaluate with the sweeps counted on the GPU: identical counts, so identical
    tpr / fpr / accuracy (reference golden) and VAL / FAR (golden + oracle)."""
    g = np.load(os.path.join(golden_dir, "verification.npz"))
    d = torch.from_numpy(g["distances"]).float().to(cuda_dev)
    lab = torch.from_numpy(g["labels"]).to(cuda_dev)
    d64 = d.cpu().numpy().astype(np.float64)          # the fp32 distances the GPU sees, as numpy would promote them
    th = np.arange(0, 30, 0.01)
    tp, fp = V.threshold_counts(d, lab, th)
    same = g["labels"].astype(bool)
    assert np.array_equal(tp, [(np.less(d64, t) & same).sum() for t in th])
    assert np.array_equal(fp, [(np.less(d64, t) & ~same).sum() for t in th])
    for target, name in ((1e-2, "1e-2"), (5e-2, "5e-2")):
        tpr, fpr, acc, val, far = V.evaluate(d, lab, far_target=target)
        otpr, ofpr, oacc = VO.evaluate_accuracy(d64, same)
        assert (tpr, fpr, acc) == (otpr, ofpr, oacc)
        assert abs(acc - float(g["ref_accuracy"])) < 1e-12 and abs(tpr - float(g["ref_tpr"])) < 1e-12
        oval, ofar, _ = VO.calculate_val(np.arange(0, 30, 0.001), d64, same, target)
        assert (val, far) == (oval, ofar)
        assert abs(val - float(g[f"val_{name}"])) < 1e-12 and abs(far - float(g[f"far_{name}"])) < 1e-12
    # degenerate inputs: no same-speaker pair -> (0, 0) as calculate_val_far returns; FAR never reaches the target -> threshold 0
    z = V.evaluate(d, torch.zeros_like(lab), far_target=1e-3)
    assert z[3] == 0.0 and z[4] == 0.0
    with pytest.raises(RuntimeError):
        V.threshold_counts(d.cpu(), lab.cpu(), th)
