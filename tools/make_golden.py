"""Generate tests/golden/*.npz from the REFERENCE ITSELF (qqueing/DeepSpeaker-pytorch's model.py, imported unmodified).

Needs a checkout of the reference project (no GPU):
    DEEPSPEAKER_REFERENCE=/path/to/DeepSpeaker-pytorch python tools/make_golden.py
The fixtures pin oracle/rescnn_oracle.py (tests/test_oracle_golden.py) and, through it, the CUDA path.
Inputs and parameters are regenerated from seeds by oracle.make_state_dict / make_input, so only
outputs are stored.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ["DEEPSPEAKER_REFERENCE"])
import model as R  # noqa: E402  (the reference's model.py)

from oracle import rescnn_oracle as O  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
NUM_CLASSES = 16
MARGIN = 0.1


def sample_idx(numel, n=16, seed=123):
    g = np.random.RandomState(seed)
    return g.randint(0, numel, size=n).astype(np.int64)


def ref_model(sd):
    m = R.DeepSpeakerModel(512, NUM_CLASSES)
    m.load_state_dict(sd)
    return m


def golden_eval():
    sd = O.make_state_dict(0, NUM_CLASSES)
    m = ref_model(sd).eval()
    out = {}
    for name, (B, T, seed, scale) in {"a": (4, 160, 0, 1.0), "b": (3, 32, 1, 10.0), "c": (2, 160, 2, 10.0)}.items():
        x = O.make_input(B, T, seed, scale)
        taps = {}
        hooks = []
        for s in range(4):
            hooks.append(getattr(m.model, f"layer{s + 1}").register_forward_hook(
                lambda mod, i, o, s=s: taps.__setitem__(3 * s + 2, o.detach().clone())))
        with torch.no_grad():
            e = m(x)
        for hk in hooks:
            hk.remove()
        out[f"{name}_cfg"] = np.array([B, T, seed, scale], dtype=np.float64)
        out[f"{name}_emb"] = e.numpy()
        for k, v in taps.items():
            flat = v.flatten()
            ix = sample_idx(flat.numel())
            out[f"{name}_tap{k}_idx"] = ix
            out[f"{name}_tap{k}_val"] = flat[ix].numpy()
            out[f"{name}_tap{k}_mean"] = np.array([flat.mean().item(), flat.abs().max().item()])
    np.savez(os.path.join(OUT, "eval_forward.npz"), **out)
    print("eval_forward.npz", {k: v.shape for k, v in out.items() if k.endswith("_emb")})


def make_triplet_embeddings(B=64, D=512, seed=5):
    g = torch.Generator().manual_seed(seed)
    nrm = lambda t: 10.0 * t / t.norm(dim=1, keepdim=True)
    a = nrm(torch.randn(B, D, generator=g))
    p = nrm(a + 0.25 * torch.randn(B, D, generator=g))
    sig = torch.linspace(0.18, 0.34, B).view(B, 1)[torch.randperm(B, generator=g)]
    n = nrm(a + sig * torch.randn(B, D, generator=g))
    return a, p, n


def golden_loss():
    a, p, n = make_triplet_embeddings()
    pd = R.PairwiseDistance(2)
    d_p = pd.forward(a, p)                                   # train_triplet.py:251
    d_n = pd.forward(a, n)                                   # :252
    allm = (d_n - d_p < MARGIN).cpu().data.numpy().flatten()  # :253
    hard = np.where(allm == 1)[0]                            # :262
    loss = R.TripletMarginLoss(MARGIN).forward(a, p, n)      # :219
    # gradients of the loss w.r.t. the embeddings (autograd through the reference's own forward)
    a2, p2, n2 = (t.clone().requires_grad_(True) for t in (a, p, n))
    R.TripletMarginLoss(MARGIN).forward(a2, p2, n2).backward()
    sel_loss = R.TripletMarginLoss(MARGIN).forward(a[hard], p[hard], n[hard])   # :275 on the selected rows
    np.savez(os.path.join(OUT, "triplet_loss.npz"), seed=np.array([64, 512, 5]), d_p=d_p.numpy(), d_n=d_n.numpy(),
             hard_idx=hard.astype(np.int64), loss=np.array(loss.item(), dtype=np.float32),
             selected_loss=np.array(sel_loss.item(), dtype=np.float32), ga=a2.grad.numpy(), gp=p2.grad.numpy(),
             gn=n2.grad.numpy())
    print("triplet_loss.npz: selected", len(hard), "of", len(allm), "loss", loss.item())


def golden_train():
    """Branch-A step (train_triplet.py:215-224) with the reference model in train mode."""
    sd = O.make_state_dict(0, NUM_CLASSES)
    m = ref_model(sd).train()
    B, T = 4, 160
    xa, xp, xn = (O.make_input(B, T, s, 3.0) for s in (10, 11, 12))
    out_a, out_p, out_n = m(xa), m(xp), m(xn)                 # :215
    loss = R.TripletMarginLoss(MARGIN).forward(out_a, out_p, out_n)   # :219
    m.zero_grad()
    loss.backward()                                           # :223
    out = {"cfg": np.array([B, T, 10, 11, 12, 3.0]), "loss": np.array(loss.item(), dtype=np.float32),
           "out_a": out_a.detach().numpy(), "out_p": out_p.detach().numpy(), "out_n": out_n.detach().numpy()}
    for k, v in m.named_parameters():
        if v.grad is None:
            continue
        gflat = v.grad.flatten()
        ix = sample_idx(gflat.numel(), 32)
        out["gnorm/" + k] = np.array(gflat.double().norm().item())
        out["gidx/" + k] = ix
        out["gval/" + k] = gflat[ix].numpy()
    for k, v in m.state_dict().items():
        if "running" in k:
            out["stat/" + k] = v.numpy()
    np.savez(os.path.join(OUT, "train_step.npz"), **out)
    print("train_step.npz: loss", loss.item(), "params with grad", sum(1 for k in out if k.startswith("gnorm/")))


def golden_branch_b(B=6, T=32, seeds=(30, 31, 32), name="branch_b_step.npz", full_head=False):
    """Branch-B step (train_triplet.py:215,251-291) with the reference model and its own forward_classifier.
    The (B=6, T=32) fixture selects 2-3 utterances (BatchNorm over 16 values per channel at stage 4: the most
    ill-conditioned shape the path can see); the (B=16, T=160) one is the well-conditioned case the 1e-3 gates use."""
    import torch.nn as nn
    sd = O.make_state_dict(0, NUM_CLASSES)
    m = ref_model(sd).train()
    xa, xp, xn = (O.make_input(B, T, s, 3.0) for s in seeds)
    g = torch.Generator().manual_seed(33)
    label_p = torch.randint(0, NUM_CLASSES, (B,), generator=g)
    label_n = torch.randint(0, NUM_CLASSES, (B,), generator=g)
    l2 = R.PairwiseDistance(2)
    out_a, out_p, out_n = m(xa), m(xp), m(xn)                                   # :215
    d_p = l2.forward(out_a, out_p)                                              # :251
    d_n = l2.forward(out_a, out_n)                                              # :252
    margin = float((d_n - d_p).median())                                        # a margin that selects about half
    allm = (d_n - d_p < margin).cpu().data.numpy().flatten()                    # :253
    hard = np.where(allm == 1)[0]                                               # :262
    sel = lambda t: torch.from_numpy(t.cpu().data.numpy()[hard])                # :265-274
    triplet = R.TripletMarginLoss(margin).forward(sel(out_a), sel(out_p), sel(out_n))   # :275
    cls_a, cls_p, cls_n = (m.forward_classifier(sel(x)) for x in (xa, xp, xn))  # :277-279
    true = torch.cat([label_p[hard], label_p[hard], label_n[hard]])             # :283
    ce = nn.CrossEntropyLoss()(torch.cat([cls_a, cls_p, cls_n]), true)          # :281-285
    loss = ce + triplet * 2.0                                                   # :287
    m.zero_grad()
    loss.backward()                                                             # :289-290
    out = {"cfg": np.array([B, T, seeds[0], seeds[1], seeds[2], 3.0, 33, margin]), "hard": hard.astype(np.int64),
           "triplet": np.array(triplet.item(), np.float32), "ce": np.array(ce.item(), np.float32),
           "loss": np.array(loss.item(), np.float32), "label_p": label_p.numpy(), "label_n": label_n.numpy()}
    for k, v in m.named_parameters():
        if v.grad is None:
            continue
        gflat = v.grad.flatten()
        ix = sample_idx(gflat.numel(), 32)
        out["gnorm/" + k] = np.array(gflat.double().norm().item())
        out["gidx/" + k] = ix
        out["gval/" + k] = gflat[ix].numpy()
        if full_head and "classifier" in k:
            out["gfull/" + k] = v.grad.numpy()
    if full_head:
        out["logits"] = torch.cat([cls_a, cls_p, cls_n]).detach().numpy()
    np.savez(os.path.join(OUT, name), **out)
    print(name, ": selected", len(hard), "of", B, "ce", ce.item(), "triplet", triplet.item(),
          "params with grad", sum(1 for k in out if k.startswith("gnorm/")))


def golden_allpairs():
    """Config 4 has no reference implementation (SURVEY §0.3): the fixture only pins the distance
    formula on pairs, computed with the reference's PairwiseDistance."""
    g = torch.Generator().manual_seed(3)
    N, D = 96, 512
    E = torch.randn(N, D, generator=g)
    E = 10.0 * E / E.norm(dim=1, keepdim=True)
    labels = (torch.arange(N) // 6).long()
    pd = R.PairwiseDistance(2)
    Dm = torch.stack([pd.forward(E[i:i + 1].expand(N, D), E) for i in range(N)])
    np.savez(os.path.join(OUT, "allpairs.npz"), seed=np.array([N, D, 3]), dist=Dm.numpy(), labels=labels.numpy())
    print("allpairs.npz", Dm.shape)


def golden_verification():
    """Best-threshold accuracy of the reference's own eval_metrics.evaluate on a fixed synthetic distance set."""
    import eval_metrics as EM  # the reference's eval_metrics.py
    g = np.random.RandomState(7)
    labels = (np.arange(400) % 2 == 0)
    distances = np.where(labels, g.normal(9.0, 2.0, 400), g.normal(13.0, 2.0, 400)).astype(np.float64)
    tpr, fpr, acc = EM.calculate_roc(np.arange(0, 30, 0.01), distances, labels)
    # evaluate()'s VAL@FAR half (eval_metrics.py:10-12) raises under current scipy (interp1d on a FAR curve with
    # duplicate x values): record that, and pin the crossing threshold with the reference's own ingredients —
    # calculate_val_far for the curve and scipy's interp1d('slinear') on the de-duplicated curve
    from scipy import interpolate
    th2 = np.arange(0, 30, 0.001)
    try:
        EM.calculate_val(th2, distances, labels, 1e-2)
        raised = ""
    except Exception as e:  # noqa: BLE001
        raised = type(e).__name__ + ": " + str(e)[:120]
    far_train = np.array([EM.calculate_val_far(t, distances, labels)[1] for t in th2])
    out = {}
    for name, target in (("1e-2", 1e-2), ("5e-2", 5e-2)):
        keep = np.concatenate(([True], np.diff(far_train) > 0))
        f = interpolate.interp1d(far_train[keep], th2[keep], kind="slinear")
        thr = float(f(target))
        val, far = EM.calculate_val_far(thr, distances, labels)
        out[f"val_threshold_{name}"] = np.array(thr)
        out[f"val_{name}"] = np.array(val)
        out[f"far_{name}"] = np.array(far)
    np.savez(os.path.join(OUT, "verification.npz"), distances=distances, labels=labels, ref_tpr=np.array(tpr),
             ref_fpr=np.array(fpr), ref_accuracy=np.array(acc), ref_calculate_val_raises=np.array(raised), **out)
    print("verification.npz: accuracy", acc, "tpr", tpr, "fpr", fpr, "| calculate_val raised:", raised or "no", "|", {k: float(v) for k, v in out.items()})


def golden_adagrad():
    """torch.optim.Adagrad with the reference's hyper-parameters (train_triplet.py:70-77,378-382) on the CPU."""
    g = torch.Generator().manual_seed(77)
    p = torch.nn.Parameter(torch.randn(4099, generator=g) * 0.05)
    p0 = p.detach().clone().numpy()
    opt = torch.optim.Adagrad([p], lr=0.1, lr_decay=1e-4, weight_decay=0.0)
    grads = []
    for it in range(6):
        gr = torch.randn(4099, generator=g) * 10.0 ** (-(it % 3))
        grads.append(gr.numpy())
        p.grad = gr.clone()
        opt.step()
    np.savez(os.path.join(OUT, "adagrad.npz"), p0=p0, grads=np.stack(grads), p_final=p.detach().numpy(),
             sum_final=opt.state[p]["sum"].numpy(), lr=np.array(0.1), lr_decay=np.array(1e-4))
    print("adagrad.npz: |p_final - p0| max", float(np.abs(p.detach().numpy() - p0).max()))


def golden_keys():
    import json
    m = R.DeepSpeakerModel(512, NUM_CLASSES)
    keys = [[k, list(v.shape)] for k, v in m.state_dict().items()]
    json.dump(keys, open(os.path.join(OUT, "state_dict_keys.json"), "w"), indent=0)
    print("state_dict_keys.json", len(keys))


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    if len(sys.argv) > 1 and sys.argv[1] == "round2":   # only the fixtures added in round 2 (the others are unchanged)
        torch.set_num_threads(8)
        golden_adagrad()
        golden_branch_b(16, 160, (40, 41, 42), "branch_b_step_b16.npz", True)
        sys.exit(0)
    golden_keys()
    torch.set_num_threads(8)
    golden_eval()
    golden_loss()
    golden_train()
    golden_branch_b()
    golden_branch_b(16, 160, (40, 41, 42), "branch_b_step_b16.npz", True)
    golden_adagrad()
    golden_verification()
    golden_allpairs()
