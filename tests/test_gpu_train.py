"""Train-mode forward (batch-statistics BN) and backward of the H100 engine vs the oracle and the
reference's golden branch-A step (train_triplet.py:215-224)."""
import os

import numpy as np
import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from oracle import rescnn_oracle as O
from tests.helpers import rel_l2

pytestmark = pytest.mark.gpu

# Tolerances.  Forward: 1e-3 (north star) with fp16 operands.
# Gradients: every backward kernel is validated in isolation against torch autograd in
# tests/test_gpu_backward_ops.py (1e-5 .. 1e-2 per op).  End to end against the fp32 reference the 16-bit stored
# activations flip the clip mask of the few elements within rounding distance of 0 or 20 (4e-4 of the elements at
# the last layer), and the untrained batch-4 network amplifies any perturbation ~2x per layer (measured with
# tools/gpu_debug_layers.py), which costs 2-10 % rel-L2 per tensor: gate on direction (cosine) and norm, report
# rel-L2.  A storage-matched fp32 oracle (oracle.forward(storage=float16)) shows the same 4-8 % on CPU.
COS_MIN = {"fp16": 0.985, "bf16": 0.90}
NORM_TOL = {"fp16": 0.03, "bf16": 0.10}


def cosine(a, b):
    return float((a.flatten().double() @ b.flatten().double()) / (a.double().norm() * b.double().norm()).clamp_min(1e-30))


def make_model(sd, dt, dev):
    m = dsk.DeepSpeakerModel(512, 16, operand_dtype=dt).to(dev)
    m.load_state_dict(sd)
    return m.train()


def run_step(m, xa, xp, xn, margin=0.1):
    out_a, out_p, out_n = m(xa), m(xp), m(xn)                      # train_triplet.py:215
    loss = dsk.TripletMarginLoss(margin).forward(out_a, out_p, out_n)   # :219
    m.zero_grad()
    loss.backward()                                                # :223
    return loss, out_a, out_p, out_n


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
def test_branch_a_step_matches_reference_golden(cuda_dev, golden_dir, dt):
    g = np.load(os.path.join(golden_dir, "train_step.npz"))
    B, T, s0, s1, s2, scale = g["cfg"]
    sd = O.make_state_dict(0, 16)
    m = make_model(sd, dt, cuda_dev)
    xa, xp, xn = (O.make_input(int(B), int(T), int(s), float(scale)).cuda() for s in (s0, s1, s2))
    loss, oa, op, on = run_step(m, xa, xp, xn)
    # train-mode BN renormalises every layer with batch statistics, which amplifies the 16-bit storage error of an
    # untrained network ~2x per layer: 0.9-1.3e-3 at batch 4-16 (eval mode, the headline path, stays at 4e-4)
    ftol = 1.5e-3 if dt == "fp16" else 1.2e-2
    for got, key in ((oa, "out_a"), (op, "out_p"), (on, "out_n")):
        ref = torch.from_numpy(g[key])
        assert ((got.detach().cpu() - ref).norm(dim=1) / ref.norm(dim=1)).max().item() < ftol, key
    # the hinge is a difference of two O(10) distances: its error is bounded relative to the distance scale
    d_scale = (oa - op).detach().norm(dim=1).mean().item()
    assert abs(loss.item() - float(g["loss"])) <= (2e-3 if dt == "fp16" else 1.5e-2) * d_scale
    # running statistics after three train-mode forwards (SURVEY §0 fact 4)
    for k, v in m.state_dict().items():
        if "running" in k:
            rt, at = (5e-3, 5e-4) if dt == "fp16" else (4e-2, 4e-3)
            assert np.allclose(v.cpu().numpy(), g["stat/" + k], rtol=rt, atol=at), k
        if "num_batches_tracked" in k:
            assert int(v.item()) == 3
    # gradients: per-tensor norm and sampled entries
    checked = 0
    for k, p in m.named_parameters():
        if "gnorm/" + k not in g:
            assert p.grad is None or "classifier" in k
            continue
        ref_norm = float(g["gnorm/" + k])
        gr = p.grad.detach().cpu()
        assert abs(gr.double().norm().item() - ref_norm) <= NORM_TOL[dt] * ref_norm + 1e-9, (k, gr.norm().item(), ref_norm)
        ix = torch.from_numpy(g["gidx/" + k])
        got_s, ref_s = gr.flatten()[ix].double(), torch.from_numpy(g["gval/" + k]).double()
        assert float(got_s @ ref_s / (got_s.norm() * ref_s.norm())) > COS_MIN[dt] - 0.05, k    # 32 sampled entries
        checked += 1
    assert checked == 38


@pytest.mark.parametrize("B,T", [(6, 160), (5, 32), (16, 48)])
def test_train_step_matches_oracle_full_gradients(cuda_dev, B, T):
    sd = O.make_state_dict(1, 16)
    m = make_model(sd, "fp16", cuda_dev)
    xa, xp, xn = (O.make_input(B, T, s, 3.0) for s in (20, 21, 22))
    loss, oa, _op, _ = run_step(m, xa.cuda(), xp.cuda(), xn.cuda())
    stats = {}
    oloss, grads, ooa, _, _ = O.triplet_step_branch_a(sd, xa, xp, xn, 0.1, stats)
    assert ((oa.detach().cpu() - ooa).norm(dim=1) / ooa.norm(dim=1)).max().item() < (1.5e-3 if T >= 160 else 3e-3)
    d_scale = (oa - _op).detach().norm(dim=1).mean().item()
    assert abs(loss.item() - oloss.item()) <= (2e-3 if T >= 160 else 6e-3) * d_scale
    for k, v in m.state_dict().items():
        if "running" in k:
            assert torch.allclose(v.cpu(), stats[k], rtol=5e-3, atol=5e-4), k
    worst_f, min_cos = 0.0, 1.0
    for k, p in m.named_parameters():
        if grads.get(k) is None:
            continue
        gr = p.grad.detach().cpu()
        rf, cs = rel_l2(gr, grads[k]), cosine(gr, grads[k])
        worst_f, min_cos = max(worst_f, rf), min(min_cos, cs)
        assert cs > COS_MIN["fp16"] and abs(gr.norm().item() / grads[k].norm().item() - 1) < NORM_TOL["fp16"], (k, cs)
    print(f"B={B} T={T}: worst grad rel-L2 vs fp32 oracle {worst_f:.3e}, min cosine {min_cos:.5f}")


def test_train_mode_without_grad_and_eval_after_train(cuda_dev):
    sd = O.make_state_dict(2, 16)
    m = make_model(sd, "fp16", cuda_dev)
    x = O.make_input(4, 32, 1, 2.0)
    with torch.no_grad():
        e = m(x.cuda())                       # train-mode BN, no graph
    st = {}
    ref = O.forward(sd, x, True, st)
    # batch 4 x T=32: stage-4 statistics come from 32 values per channel, the most ill-conditioned case
    assert ((e.cpu() - ref).norm(dim=1) / ref.norm(dim=1)).max().item() < 3e-3
    m.eval()                                  # eval fold must pick up the updated running stats
    sd2 = dict(sd)
    sd2.update(st)
    with torch.no_grad():
        e2 = m(x.cuda()).cpu()
        ref2 = O.forward(sd2, x)
    assert ((e2 - ref2).norm(dim=1) / ref2.norm(dim=1)).max().item() < 1e-3


def test_optimizer_step_is_picked_up(cuda_dev):
    """Adagrad step as in train_triplet.py:378-382, then a second forward must use the new weights."""
    sd = O.make_state_dict(3, 16)
    m = make_model(sd, "fp16", cuda_dev)
    opt = torch.optim.Adagrad(m.parameters(), lr=0.01, lr_decay=1e-4, weight_decay=0.0)
    xa, xp, xn = (O.make_input(4, 32, s, 3.0).cuda() for s in (1, 2, 3))
    l0, *_ = run_step(m, xa, xp, xn, margin=5.0)      # a margin that keeps every triplet active
    opt.step()
    l1, *_ = run_step(m, xa, xp, xn, margin=5.0)
    assert torch.isfinite(l0) and torch.isfinite(l1) and abs(l0.item() - l1.item()) > 0
    assert m.model.classifier.weight.grad is None          # SURVEY §0 fact 5


def test_branch_b_step_matches_reference_golden(cuda_dev, golden_dir):
    """train_triplet.py:215,251-291 with the drop-in classes: selection on the device, second forward through
    forward_classifier, cross-entropy + 2 x (constant) triplet term, backward.  The reference's own selection
    indices are used so that both sides differentiate the same samples."""
    g = np.load(os.path.join(golden_dir, "branch_b_step.npz"))
    B, T, s0, s1, s2, scale, lseed, margin = g["cfg"]
    sd = O.make_state_dict(0, 16)
    m = make_model(sd, "fp16", cuda_dev)
    xa, xp, xn = (O.make_input(int(B), int(T), int(s), float(scale)).cuda() for s in (s0, s1, s2))
    label_p, label_n = torch.from_numpy(g["label_p"]).cuda(), torch.from_numpy(g["label_n"]).cuda()
    out_a, out_p, out_n = m(xa), m(xp), m(xn)                                            # :215
    l2 = dsk.PairwiseDistance(2)
    d_p, d_n = l2.forward(out_a, out_p), l2.forward(out_a, out_n)                        # :251-252
    idx, cnt = dsk.select_hard_triplets(d_p, d_n, float(margin))                         # :253-262 on the device
    k = int(cnt.item())
    assert 0 < k <= int(B)
    # the margin is the median of d_n - d_p, so the engine's fp16-level distance error may move a boundary sample
    assert len(set(idx[:k].tolist()) ^ set(g["hard"].tolist())) <= 2
    h = torch.from_numpy(g["hard"]).cuda()
    sel = lambda t: t.detach()[h]                                                        # :265-274 (detached)
    triplet = dsk.TripletMarginLoss(float(margin)).forward(sel(out_a), sel(out_p), sel(out_n))   # :275
    cls = [m.forward_classifier(x[h].contiguous()) for x in (xa, xp, xn)]               # :277-279
    true = torch.cat([label_p[h], label_p[h], label_n[h]])                               # :283
    ce = dsk.CrossEntropyLoss()(torch.cat(cls), true)                                    # :281-285 (repo kernels)
    loss = ce + triplet * 2.0                                                            # :287
    m.zero_grad()
    loss.backward()                                                                      # :289-290
    # batch of 2 selected utterances at T=32: BatchNorm statistics over 16 values per channel at stage 4 — the most
    # ill-conditioned shape the path can see, hence the loose forward gates
    assert abs(ce.item() - float(g["ce"])) <= 5e-2 * float(g["ce"])
    assert abs(triplet.item() - float(g["triplet"])) <= 3e-2 * max(1.0, float(g["triplet"]))
    checked = 0
    for kname, p in m.named_parameters():
        if "gnorm/" + kname not in g:
            continue
        assert p.grad is not None, kname
        ref_norm = float(g["gnorm/" + kname])
        assert abs(p.grad.double().norm().item() - ref_norm) <= 0.15 * ref_norm + 1e-9, (kname, p.grad.norm().item(), ref_norm)
        checked += 1
    assert checked == 40 and m.model.classifier.weight.grad is not None


def test_branch_b_step_b16_matches_reference_golden(cuda_dev, golden_dir):
    """The well-conditioned branch-B fixture (16 triplets, T=160, 7 selected): classifier logits, cross-entropy and the
    classifier gradients through the repo's own GEMM / log-softmax kernels at the north star's 1e-3."""
    g = np.load(os.path.join(golden_dir, "branch_b_step_b16.npz"))
    B, T, s0, s1, s2, scale, lseed, margin = g["cfg"]
    sd = O.make_state_dict(0, 16)
    m = make_model(sd, "fp16", cuda_dev)
    xa, xp, xn = (O.make_input(int(B), int(T), int(s), float(scale)).cuda() for s in (s0, s1, s2))
    label_p, label_n = torch.from_numpy(g["label_p"]).cuda(), torch.from_numpy(g["label_n"]).cuda()
    out_a, out_p, out_n = m(xa), m(xp), m(xn)                                            # :215
    l2 = dsk.PairwiseDistance(2)
    d_p, d_n = l2.forward(out_a, out_p), l2.forward(out_a, out_n)                        # :251-252
    idx, cnt = dsk.select_hard_triplets(d_p, d_n, float(margin))                         # :253-262
    k = int(cnt.item())
    assert len(set(idx[:k].tolist()) ^ set(g["hard"].tolist())) <= 2                     # margin = median of d_n - d_p
    h = torch.from_numpy(g["hard"]).cuda()
    sel = lambda t: t.detach()[h]
    triplet = dsk.TripletMarginLoss(float(margin)).forward(sel(out_a), sel(out_p), sel(out_n))   # :275
    cls = torch.cat([m.forward_classifier(x[h].contiguous()) for x in (xa, xp, xn)])    # :277-279
    true = torch.cat([label_p[h], label_p[h], label_n[h]])                               # :283
    ce = dsk.CrossEntropyLoss()(cls, true)                                               # :281-285
    loss = ce + triplet * 2.0                                                            # :287
    m.zero_grad()
    loss.backward()                                                                      # :289-290
    ref_logits = torch.from_numpy(g["logits"])
    assert (cls.detach().cpu() - ref_logits).abs().max().item() <= 2e-3 * ref_logits.abs().max().item()
    assert abs(ce.item() - float(g["ce"])) <= 1e-3 * float(g["ce"])
    assert abs(triplet.item() - float(g["triplet"])) <= 2e-3 * 10.0      # distances are O(10): 1e-3 relative to them
    for kname in ("model.classifier.weight", "model.classifier.bias"):
        got, ref = dict(m.named_parameters())[kname].grad.cpu(), torch.from_numpy(g["gfull/" + kname])
        assert rel_l2(got, ref) < 5e-3, (kname, rel_l2(got, ref))
    checked = 0
    for kname, p in m.named_parameters():
        if "gnorm/" + kname not in g:
            continue
        ref_norm = float(g["gnorm/" + kname])
        assert abs(p.grad.double().norm().item() - ref_norm) <= 0.05 * ref_norm + 1e-9, (kname, p.grad.norm().item(), ref_norm)
        checked += 1
    assert checked == 40


def test_forward_triplet_is_bit_identical_to_three_sequential_calls(cuda_dev):
    """forward_triplet (three train forwards + their backwards in flight on three streams, running statistics committed in
    call order) against model(a), model(p), model(n) called one after the other (train_triplet.py:215): same bits for the
    embeddings, the running statistics, num_batches_tracked and every gradient."""
    sd = O.make_state_dict(4, 16)
    xs = [O.make_input(12, 64, s, 3.0).cuda() for s in (7, 8, 9)]
    res = []
    for fused in (False, True):
        m = make_model(sd, "fp16", cuda_dev)
        for rep in range(2):                         # twice: contexts are recycled, running stats keep moving
            outs = m.forward_triplet(*xs) if fused else (m(xs[0]), m(xs[1]), m(xs[2]))
            loss = dsk.TripletMarginLoss(0.1).forward(*outs)
            m.zero_grad()
            loss.backward()
        torch.cuda.synchronize()
        res.append(([o.detach().clone() for o in outs], {k: v.clone() for k, v in m.state_dict().items()},
                    {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}, loss.detach().clone()))
    (o0, s0, g0, l0), (o1, s1, g1, l1) = res
    assert torch.equal(l0, l1)
    for a, b in zip(o0, o1):
        assert torch.equal(a, b)
    for k in s0:
        assert torch.equal(s0[k], s1[k]), k
    assert len(g0) == 38
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    # without autograd (train-mode BN under no_grad) the contexts are committed and released
    m = make_model(sd, "fp16", cuda_dev)
    with torch.no_grad():
        e = m.forward_triplet(*xs)
    m2 = make_model(sd, "fp16", cuda_dev)
    with torch.no_grad():
        e2 = (m2(xs[0]), m2(xs[1]), m2(xs[2]))
    for a, b in zip(e, e2):
        assert torch.equal(a, b)
    for k, v in m.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k]), k
    m.eval()
    with torch.no_grad():
        ev = m.forward_triplet(*xs)
        assert torch.equal(ev[1], m(xs[1]))


def test_forward_triplet_accumulates_into_an_optimizer_bucket_like_autograd(cuda_dev):
    """With FusedAdagrad (or GradBucket) every p.grad is a view of one flat bucket; TripletForwardFn then adds its summed
    gradients into the bucket with one multi-tensor add and returns no per-parameter gradients.  Must give the bits
    autograd's own accumulation gives for three sequential calls - also on top of a non-zero bucket (two backwards
    without zero_grad) and after the views were dropped (module.zero_grad() -> falls back to returning gradients)."""
    sd = O.make_state_dict(6, 16)
    xs = [O.make_input(10, 64, s, 3.0).cuda() for s in (41, 42, 43)]
    res = []
    for fused in (False, True):
        m = make_model(sd, "fp16", cuda_dev)
        opt = dsk.FusedAdagrad(m.parameters(), lr=1e-3)
        opt.zero_grad()
        for rep in range(2):                         # second backward accumulates on top of the first
            outs = m.forward_triplet(*xs) if fused else (m(xs[0]), m(xs[1]), m(xs[2]))
            dsk.TripletMarginLoss(0.1).forward(*outs).backward()
        torch.cuda.synchronize()
        assert all(p.grad is p._dsk_bucket_grad for p in opt.params)
        assert m._engine.bucket_accumulations == (2 if fused else 0)
        res.append(opt.flat_grad.clone())
        opt.step()
        res.append(opt.flat_param.clone())
    assert torch.equal(res[0], res[2]) and torch.equal(res[1], res[3])
    assert res[0].abs().max() > 0
    # torch.autograd.grad captures gradients instead of accumulating them: the bucket must stay untouched
    before = opt.flat_grad.clone()
    path = [p for p in opt.params if p.grad is not None][:38]
    got = torch.autograd.grad(dsk.TripletMarginLoss(0.1).forward(*m.forward_triplet(*xs)), path, allow_unused=True)
    assert torch.equal(opt.flat_grad, before) and sum(g is not None and bool(g.abs().max() > 0) for g in got) >= 36
    assert m._engine.bucket_accumulations == 2
    m.zero_grad()                                    # set_to_none: the bucket views are gone -> ordinary autograd path
    dsk.TripletMarginLoss(0.1).forward(*m.forward_triplet(*xs)).backward()
    assert sum(p.grad is not None for p in m.parameters()) == 38


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
def test_training_weight_repack_writes_the_same_operand_images(cuda_dev, dt):
    """dsk_load_weights_train (one table-driven launch per step, only the images the training path reads) against the full
    dsk_load_weights (per-layer pack kernels): a train-mode forward + backward must give the same bits with either, and an
    eval forward on a handle that only holds the training images is refused."""
    import ctypes
    from deepspeaker_pytorch_b200 import _lib as L
    sd = O.make_state_dict(8, 16)
    xs = [O.make_input(6, 64, s, 3.0).cuda() for s in (51, 52, 53)]
    m = make_model(sd, dt, cuda_dev)

    def step():
        outs = m.forward_triplet(*xs)
        m.zero_grad()
        dsk.TripletMarginLoss(0.1).forward(*outs).backward()
        torch.cuda.synchronize()
        return [o.detach().clone() for o in outs], {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}

    o_train, g_train = step()                                   # sync_weights(train) -> dsk_load_weights_train
    eng = m._engine
    x0, emb = xs[0].contiguous(), torch.empty(6, 512, device="cuda")
    rc = eng.lib.dsk_rescnn_forward(eng.handle, x0.data_ptr(), 6, 64, emb.data_ptr(), 0, L.cur_stream())
    assert rc != 0 and b"dsk_load_weights_train" in eng.lib.dsk_last_error()
    L.check(eng.lib.dsk_load_weights(eng.handle, ctypes.byref(eng._wstruct), L.cur_stream()), "dsk_load_weights")
    o_full, g_full = step()                                     # parameter versions unchanged: no repack in between
    for a, b in zip(o_train, o_full):
        assert torch.equal(a, b)
    assert len(g_train) == 38
    for k in g_train:
        assert torch.equal(g_train[k], g_full[k]), k
    m.eval()                                                    # the shim reloads everything for an eval forward
    with torch.no_grad():
        e = m(xs[0])
    assert torch.isfinite(e).all() and abs(float(e.norm(dim=1).mean()) - 10.0) < 1e-3


def test_train_step_helper_runs_both_branches_like_the_oracle(cuda_dev, golden_dir):
    """steps.train_step (train_triplet.py:208-299 restated with device-side selection) against the oracle's branch-B step
    on the reference golden's configuration, then a branch-A step through the same helper."""
    g = np.load(os.path.join(golden_dir, "branch_b_step_b16.npz"))
    B, T, s0, s1, s2, scale, lseed, margin = g["cfg"]
    sd = O.make_state_dict(0, 16)
    m = make_model(sd, "fp16", cuda_dev)
    opt = dsk.FusedAdagrad(m.parameters(), lr=1e-3, lr_decay=1e-4)
    xa, xp, xn = (O.make_input(int(B), int(T), int(s), float(scale)).cuda() for s in (s0, s1, s2))
    label_p, label_n = torch.from_numpy(g["label_p"]).cuda(), torch.from_numpy(g["label_n"]).cuda()
    r = dsk.train_step(m, opt, xa, xp, xn, label_p, label_n, margin=float(margin), epoch=1, min_softmax_epoch=2)
    assert r is not None and r["selected"] == len(r["hard"])
    assert len(set(r["hard"].tolist()) ^ set(g["hard"].tolist())) <= 2          # margin = median of d_n - d_p
    if set(r["hard"].tolist()) == set(g["hard"].tolist()):
        assert abs(r["ce"].item() - float(g["ce"])) <= 1e-3 * float(g["ce"])
        assert abs(r["triplet"].item() - float(g["triplet"])) <= 2e-3 * 10.0
    assert opt.step_count == 1 and m.model.classifier.weight.grad is not None
    # nothing selected -> None, no optimizer step (train_triplet.py:263-264)
    r0 = dsk.train_step(m, opt, xa, xp, xn, label_p, label_n, margin=-1e9, epoch=1)
    assert r0 is None and opt.step_count == 1
    # branch A through the same helper
    rA = dsk.train_step(m, opt, xa, xp, xn, label_p, label_n, margin=0.1, epoch=3, min_softmax_epoch=2)
    assert rA["ce"] is None and rA["selected"] == int(B) and opt.step_count == 2 and torch.isfinite(rA["loss"])
    with pytest.raises(RuntimeError):
        dsk.train_step(m.eval(), opt, xa, xp, xn, label_p, label_n, margin=0.1, epoch=3)


@pytest.mark.parametrize("shrink", [1e-2, 1e-4, 1e-6])
def test_fp16_backward_survives_small_gradients(cuda_dev, shrink):
    """fp16 gradient tensors are multiplied by a power-of-two loss scale inside the backward.  Round 1 used a static scale
    (2^(9 + log2 B)) that no test stressed: late in training the loss - and every gradient with it - is orders of
    magnitude smaller than in a fresh network, and a backward that underflows stops being linear in the incoming
    gradient.  The scale is now chosen per backward on the device from max|dL/d(fc output)| (loss_scale_kernel):
    shrinking the loss by 1e-2 ... 1e-6 must shrink every parameter gradient by exactly that factor (to fp16 rounding).
    The same step with the scale pinned to round 1's static value shows what the dynamic choice buys."""
    sd = O.make_state_dict(5, 16)
    xs = [O.make_input(16, 64, s, 3.0).cuda() for s in (31, 32, 33)]

    def grads_of(mult, scale=None):
        m = make_model(sd, "fp16", cuda_dev)
        if scale is not None:
            m(xs[0])                                      # creates the engine
            m._engine.set_loss_scale(scale)
        outs = m.forward_triplet(*xs)
        loss = dsk.TripletMarginLoss(0.5).forward(*outs) * mult
        m.zero_grad()
        loss.backward()
        return {k: p.grad.detach().double().cpu() / mult for k, p in m.named_parameters() if p.grad is not None}

    ref = grads_of(1.0)
    small = grads_of(shrink)
    worst = max((rel_l2(small[k], ref[k]), k) for k in ref)
    static = grads_of(shrink, scale=2.0 ** 13)            # round 1's rule at batch 16
    worst_s = max((rel_l2(static[k], ref[k]), k) for k in ref)
    print(f"loss x {shrink:g}: worst gradient rel-L2 vs the unshrunk step: dynamic scale {worst[0]:.2e} ({worst[1]}), "
          f"static 2^13 {worst_s[0]:.2e} ({worst_s[1]})")
    assert worst[0] < 2e-3, worst
