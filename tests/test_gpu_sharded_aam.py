"""The class-sharded AAM-softmax on the GPU, R ranks emulated in one process through one handle: cos, sub and top
bit-identical to the whole op, the loss and gradients against fp64, every output bit-identical across 128-aligned
class splits (gE within 1e-6), determinism and independence from other ops' calls, NaN containment as in the whole op,
bad ranges, a class count above the whole op's cap, the step at world size 1, and with >= 2 GPUs (NCCL) the sharded
step against the single-device step on the gathered batch."""
import os
import socket
import zlib

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import engine as EN
from deepspeaker_pytorch_b200 import parallel as P
from deepspeaker_pytorch_b200 import train as TR
from oracle import aam_softmax_oracle as A
from oracle import rescnn_oracle as O
from oracle import subcentre_aam_oracle as S
from tests.test_gpu_aam_softmax import _row_rel

pytestmark = pytest.mark.gpu

M, SC, TM = 0.2, 30.0, 0.1


def _case(N, C, K, D=512):
    g = torch.Generator().manual_seed(zlib.crc32(f"shard{N}x{C}x{K}x{D}".encode()))
    E = torch.randn(N, D, generator=g)
    E = 10.0 * E / E.norm(dim=1, keepdim=True)
    W = torch.randn(C * K, D, generator=g) / D ** 0.5
    return E.cuda(), W.cuda(), torch.randint(0, C, (N,), generator=g).cuda()


def _splits(C):
    """R = 1, 2, 4, 8 (class_shards) and an uneven 128-aligned split of four ranks (one block, a third, the rest but
    the last partial block, the last block)."""
    out = [P.class_shards(C, R) for R in (1, 2, 4, 8)]
    nb = -(-C // 128)
    b = max(2, nb // 3)
    c = max(b + 1, nb - 1)
    out.append([(0, 128), (128, 128 * b), (128 * b, 128 * c), (128 * c, C)])
    return out


def run_split(E, W, y, K, topk, ranges, grad=1.0, m=M, s=SC, tm=TM):
    """The sharded op over the class ranges, R = len(ranges) ranks emulated in lockstep (stage by stage, as
    ShardedAAMSoftmaxLoss.forward_stages / backward_stages run them) -> dict of cos, sub, top (concatenated over the
    shards), loss, lse, row_loss, gE, gW."""
    R, (N, D), C = len(ranges), E.shape, W.shape[0] // K
    n = N // R
    nb = max(-(-(c1 - c0) // 128) for c0, c1 in ranges)
    Ws = [W[c0 * K:c1 * K].contiguous() for c0, c1 in ranges]
    st1 = [EN.aam_shard_cos(E, Wr, y, C, c0, c1, K, topk) for Wr, (c0, c1) in zip(Ws, ranges)]
    keys = P.emulated_gather([k for _, _, k in st1])[0] if topk else None
    st2 = [EN.aam_shard_merge(c, y, keys, R, C, c0, c1, topk, m, s, tm) for (c, _, _), (c0, c1) in zip(st1, ranges)]
    maxima = P.emulated_gather([ml for _, _, ml in st2])[0]
    st3 = [EN.aam_shard_partials(c, y, thr, maxima, R, C, c0, c1, topk, nb, m, s, tm)
           for (c, _, _), (_, thr, _), (c0, c1) in zip(st1, st2, ranges)]
    rec = P.emulated_gather([r for _, r in st3])[0]
    fin = [EN.aam_shard_finish(rec, mm, y, R, C, nb) for mm, _ in st3]
    for f in fin[1:]:
        assert all(_nan_eq(a, b) for a, b in zip(f, fin[0]))              # every rank finishes with the same bits
    loss, lse, row_loss, den = fin[0]
    gl = torch.full((), float(grad), device="cuda")
    bwd = [EN.aam_shard_backward(E, Wr, y, c, sb, thr, mm, den, C, c0, c1, m, s, K, topk, tm, gl)
           for Wr, (c, sb, _), (_, thr, _), (mm, _), (c0, c1) in zip(Ws, st1, st2, st3, ranges)]
    recv = P.emulated_all_to_all([p for _, p in bwd])
    gE = torch.cat([EN.aam_shard_backward_rows(E[r * n:(r + 1) * n].contiguous(), recv[r], R) for r in range(R)])
    tops = [t for t, _, _ in st2]
    assert all(_eq(t, tops[0]) for t in tops)
    return dict(cos=torch.cat([c for c, _, _ in st1], 1), sub=None if K == 1 else torch.cat([b for _, b, _ in st1], 1),
                top=tops[0], loss=loss.reshape(()), lse=lse, row_loss=row_loss, gE=gE, gW=torch.cat([g for g, _ in bwd]))


def _eq(a, b):
    if a is None or b is None:
        return a is None and b is None
    return torch.equal(a, b)


def _nan_eq(a, b):
    """Bit equality with NaN == NaN (NaN payloads aside)."""
    na, nb_ = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb_) and torch.equal(a[~na], b[~nb_])


def _whole(E, W, y, K, topk, grad=1.0):
    _, _, _, loss, cos, lse, sub, top = EN.aam_softmax_sc(E, W, y, M, SC, K, topk, TM)
    gE, gW = EN.aam_softmax_sc_backward(E, W, y, cos, lse, sub, top, M, SC, K, topk, TM,
                                        torch.full((), float(grad), device="cuda"))
    return dict(loss=loss.reshape(()), cos=cos, lse=lse, sub=sub, top=top, gE=gE, gW=gW)


def _ref64(E, W, y, K, topk, cos, sub, top):
    """fp64 on the GPU with cos / sub / top pinned (subcentre_aam_oracle's forward and backward) -> loss, lse, gE, gW."""
    N, C = cos.shape
    e, ne = A._normalize(E.double())
    w, nw = A._normalize(W.double())
    c = cos.double()
    ar = torch.arange(N, device=E.device)
    lg = SC * c.clone()
    if topk:
        inT = torch.zeros(N, C, dtype=torch.bool, device=E.device)
        inT[ar[:, None], top.long()] = True
        lg[inT] = SC * S.psi(c[inT], TM)
    lg[ar, y] = SC * A.phi(c[ar, y], M)
    lse = torch.logsumexp(lg, 1)
    loss = (lse - lg[ar, y]).sum() / N
    d = torch.softmax(lg, 1)
    d[ar, y] -= 1.0
    d *= SC / N
    if topk:
        d[inT] *= S.dpsi(c[inT], TM)
    d[ar, y] *= A.dphi(c[ar, y], M)
    sb = torch.zeros(N, C, dtype=torch.long, device=E.device) if sub is None else sub.long()
    dx = torch.zeros(N, C * K, dtype=torch.float64, device=E.device)
    dx[ar[:, None], torch.arange(C, device=E.device)[None, :] * K + sb] = d
    del d
    ge, gw = dx @ w, dx.T @ e
    gE = (ge - e * (e * ge).sum(1, keepdim=True)) / ne
    gW = (gw - w * (w * gw).sum(1, keepdim=True)) / nw
    return loss, lse, gE, gW


SHAPES = [(384, 1211), (1024, 3 * 5994), (3072, 3 * 5994)]
CASES = [(sh, K, t) for sh in SHAPES for K in (1, 3) for t in (0, 5, 64)]


@pytest.mark.parametrize("shape,K,topk", CASES, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_against_whole_op_and_fp64_and_across_splits(cuda_dev, shape, K, topk):
    N, C = shape
    E, W, y = _case(N, C, K)
    ref = _whole(E, W, y, K, topk)
    base = None
    for ranges in _splits(C):
        out = run_split(E, W, y, K, topk, ranges)
        assert torch.equal(out["cos"], ref["cos"]) and _eq(out["sub"], ref["sub"]) and _eq(out["top"], ref["top"]), \
            ranges
        if base is None:
            base = out
            oloss, olse, oE, oW = _ref64(E, W, y, K, topk, ref["cos"], ref["sub"], ref["top"])
            assert abs(out["loss"].item() - oloss.item()) <= 1e-5 * max(abs(oloss.item()), 1.0)
            e_lse = float((out["lse"].double() - olse).abs().max() / olse.abs().max())
            eE, eW = _row_rel(out["gE"], oE.cpu()), _row_rel(out["gW"], oW.cpu())
            assert e_lse <= 1e-6 and eE <= 1e-5 and eW <= 1e-5, (e_lse, eE, eW)
            print(f"\n{shape} K {K} topk {topk}: loss {out['loss'].item():.6f} vs fp64 {oloss.item():.6f} "
                  f"(whole op {ref['loss'].item():.6f}), lse {e_lse:.1e}, gE {eE:.2e}, gW {eW:.2e}")
            continue
        for k in ("lse", "row_loss", "loss", "gW"):
            assert torch.equal(out[k], base[k]), (k, ranges)
        rel = float((out["gE"] - base["gE"]).double().norm() / base["gE"].double().norm())
        assert rel <= 1e-6, (ranges, rel)


def test_heads_in_lockstep_are_the_stages(cuda_dev):
    """ShardedAAMSoftmaxLoss heads with shard=(r, R), driven through train.run_lockstep and the emulated exchanges,
    give the bits of the stage-by-stage driver; R = 1 through forward() / autograd gives the R = 1 bits."""
    N, C, K, topk, R = 512, 1211, 3, 5, 4
    E, W, y = _case(N, C, K)
    n = N // R
    heads = [P.ShardedAAMSoftmaxLoss(W, M, SC, subcentres=K, topk=topk, topk_margin=TM, shard=(r, R)) for r in range(R)]
    sts = TR.run_lockstep([h.forward_stages(E[r * n:(r + 1) * n], y) for r, h in enumerate(heads)], P.emulated_gather)
    gl = torch.full((), 2.0, device="cuda")
    outs = TR.run_lockstep([h.backward_stages(st, gl) for h, st in zip(heads, sts)], P.emulated_all_to_all)
    ref = run_split(E, W, y, K, topk, P.class_shards(C, R), grad=2.0)
    assert all(torch.equal(st.loss.reshape(()), ref["loss"]) for st in sts)
    assert torch.equal(torch.cat([st.cos for st in sts], 1), ref["cos"])
    assert torch.equal(torch.cat([g for g, _ in outs]), ref["gE"]) and torch.equal(torch.cat([w for _, w in outs]),
                                                                                     ref["gW"])
    head = P.ShardedAAMSoftmaxLoss(W, M, SC, subcentres=K, topk=topk, topk_margin=TM)
    Ein = E.clone().requires_grad_(True)
    loss = head(Ein, y)
    loss.backward(gl)
    one = run_split(E, W, y, K, topk, [(0, C)], grad=2.0)
    assert torch.equal(loss.detach(), one["loss"]) and torch.equal(Ein.grad, one["gE"])
    assert torch.equal(head.weight.grad, one["gW"]) and torch.equal(head.full_weight(), W)


def test_deterministic_and_independent_of_other_calls(cuda_dev):
    from tests.test_gpu_ge2e import _case as ge2e_case, _csr, _scalar

    N, C, K, topk = 1024, 3 * 5994, 3, 5
    E, W, y = _case(N, C, K)
    splits = [P.class_shards(C, 4), [(0, 128), (128, 5120), (5120, C)]]
    first = [run_split(E, W, y, K, topk, r) for r in splits]
    E2, W2, y2 = _case(384, 1211, 3)
    EN.aam_softmax_sc(E2, W2, y2, M, SC, 3, 64, TM)
    Eg, lg = ge2e_case([4] * 64, 512, "norm10", 3)
    csr, V = _csr(lg)
    EN.ge2e(Eg.cuda(), csr, V, _scalar(10.0), _scalar(-5.0), "softmax")
    EN.cohort_stats(E[:100], E2, 50)
    for r, f in zip(splits, first):
        again = run_split(E, W, y, K, topk, r)
        for k in f:
            assert _eq(again[k], f[k]), k


def test_nan_row_and_nan_weight_row_as_the_whole_op(cuda_dev):
    N, C, K, topk = 256, 1211, 3, 5
    E, W, y = _case(N, C, K)
    ranges = P.class_shards(C, 4)
    clean = run_split(E, W, y, K, topk, ranges)
    bad = E.clone()
    bad[17, 5] = float("nan")
    out, ref = run_split(bad, W, y, K, topk, ranges), _whole(bad, W, y, K, topk)
    assert _nan_eq(out["cos"], ref["cos"]) and torch.equal(out["sub"], ref["sub"]) and torch.equal(out["top"], ref["top"])
    for k in ("lse", "gE", "gW"):
        assert torch.equal(torch.isnan(out[k]), torch.isnan(ref[k])), k
    assert torch.isnan(out["loss"]) and torch.isnan(out["row_loss"][17])
    keep = torch.arange(N, device="cuda") != 17
    for k in ("lse", "row_loss"):
        assert torch.equal(out[k][keep], clean[k][keep]), k
    rel = float((out["gE"][keep] - clean["gE"][keep]).double().norm() / clean["gE"][keep].double().norm())
    assert rel == 0.0 or rel <= 1e-6
    Wb = W.clone()
    Wb[700 * K + 1, 3] = float("nan")                      # class 700 (on rank 2 of 4), sub-centre 1
    out, ref = run_split(E, Wb, y, K, topk, ranges), _whole(E, Wb, y, K, topk)
    assert _nan_eq(out["cos"], ref["cos"]) and torch.equal(out["sub"], ref["sub"]) and torch.equal(out["top"], ref["top"])
    for k in ("loss", "lse", "gE", "gW"):
        assert torch.equal(torch.isnan(out[k]), torch.isnan(ref[k])), k


def test_bad_ranges_are_rejected(cuda_dev):
    E, W, y = _case(64, 1000, 1, 64)
    for c0, c1, K, topk, C in ((64, 1000, 1, 0, 1000), (0, 1001, 1, 0, 1000), (128, 128, 1, 0, 1000),
                               (256, 128, 1, 0, 1000), (0, 200, 1, 0, 1000), (-128, 128, 1, 0, 1000),
                               (0, 1000, 1, 65, 1000), (0, 128, 1, 5, 5), (0, 65536, 2, 0, 70000),
                               (0, 1000, 17, 0, 1000)):
        Wr = torch.randn(max(c1 - c0, 1) * K, 64, device="cuda")
        with pytest.raises(RuntimeError):
            EN.aam_shard_cos(E, Wr, y, C, c0, c1, K, topk)
    cos = torch.zeros(64, 1000, device="cuda")
    with pytest.raises(RuntimeError):
        EN.aam_shard_partials(cos, y, None, torch.zeros(64, device="cuda"), 1, 1000, 0, 1000, 0, 7, M, SC, TM)
    with pytest.raises(RuntimeError):
        EN.aam_shard_merge(cos, y, None, 1, 1000, 0, 1000, 0, -0.1, SC, TM)


def test_engine_wrappers_check_their_tensors(cuda_dev):
    """The C ABI sees pointers only: a full weight for a shard, a strided view, a wrong dtype or device, or state of
    the wrong shape is refused in Python before any launch."""
    N, C, K, topk = 64, 1000, 3, 5
    E, W, y = _case(N, C, K, 64)
    c0, c1 = 128, 512
    Wr = W[c0 * K:c1 * K].contiguous()
    cos, sub, keys = EN.aam_shard_cos(E, Wr, y, C, c0, c1, K, topk)
    for args in ((E, W, y), (E.t().contiguous().t(), Wr, y), (E.double(), Wr, y), (E, Wr, y.int()), (E, Wr, y.cpu()),
                 (E, Wr[:-3], y), (E[:, :32], Wr, y)):
        with pytest.raises(RuntimeError):
            EN.aam_shard_cos(*args, C, c0, c1, K, topk)
    with pytest.raises(RuntimeError):                          # cos of another range
        EN.aam_shard_merge(cos[:, :100].contiguous(), y, keys.reshape(-1), 1, C, c0, c1, topk, M, SC, TM)
    with pytest.raises(RuntimeError):                          # keys of 2 ranks for R = 1
        EN.aam_shard_merge(cos, y, keys.repeat(2, 1), 1, C, c0, c1, topk, M, SC, TM)
    top, thr, mloc = EN.aam_shard_merge(cos, y, keys, 1, C, c0, c1, topk, M, SC, TM)
    with pytest.raises(RuntimeError):                          # maxima of 1 rank for R = 2
        EN.aam_shard_partials(cos, y, thr, mloc, 2, C, c0, c1, topk, 3, M, SC, TM)
    m, rec = EN.aam_shard_partials(cos, y, thr, mloc, 1, C, c0, c1, topk, 3, M, SC, TM)
    with pytest.raises(RuntimeError):                          # records of another width
        EN.aam_shard_finish(rec, m, y, 1, C, 4)
    den = torch.ones(N, 2, device="cuda")                    # (S, S_other) stand-ins: only the shapes are checked
    gl = torch.ones((), device="cuda")
    with pytest.raises(RuntimeError):                          # the full weight for the shard
        EN.aam_shard_backward(E, W, y, cos, sub, thr, m, den, C, c0, c1, M, SC, K, topk, TM, gl)
    with pytest.raises(RuntimeError):                          # sub missing at K = 3
        EN.aam_shard_backward(E, Wr, y, cos, None, thr, m, den, C, c0, c1, M, SC, K, topk, TM, gl)
    gW, part = EN.aam_shard_backward(E, Wr, y, cos, sub, thr, m, den, C, c0, c1, M, SC, K, topk, TM, gl)
    with pytest.raises(RuntimeError):
        EN.aam_shard_backward_rows(E, part[:10], 1)


def test_above_the_whole_ops_class_cap(cuda_dev):
    N, C, K, topk = 256, 100000, 1, 5
    E, W, y = _case(N, C, K)
    with pytest.raises(RuntimeError):
        EN.aam_softmax_sc(E, W, y, M, SC, K, topk, TM)
    ranges = P.class_shards(C, 2)
    out = run_split(E, W, y, K, topk, ranges)
    other = run_split(E, W, y, K, topk, P.class_shards(C, 4))           # 782 blocks per row through the finish
    for k in ("cos", "top", "lse", "row_loss", "loss", "gW"):
        assert torch.equal(other[k], out[k]), k
    e, _ = A._normalize(E.double())
    w, _ = A._normalize(W.double())
    c64 = e @ w.T
    dc = float((out["cos"].double() - c64).abs().max())
    assert dc <= 1e-6, dc
    sel = c64.clone()
    sel[torch.arange(N, device="cuda"), y] = -2.0
    tv = sel.topk(topk + 1, dim=1).values
    clear = (tv[:, :-1] - tv[:, 1:]).min(1).values > 4e-6
    assert torch.equal(out["top"].long()[clear].sort(1).values, sel.topk(topk, dim=1).indices[clear].sort(1).values)
    oloss, olse, oE, oW = _ref64(E, W, y, K, topk, out["cos"], None, out["top"])
    eE, eW = _row_rel(out["gE"], oE.cpu()), _row_rel(out["gW"], oW.cpu())
    assert abs(out["loss"].item() - oloss.item()) <= 1e-5 * max(oloss.item(), 1.0) and eE <= 1e-5 and eW <= 1e-5
    print(f"\nC = {C}, R = 2: |dcos| {dc:.2e}, loss {out['loss'].item():.6f} vs {oloss.item():.6f}, gE {eE:.2e}, "
          f"gW {eW:.2e}")


def _flat_rel(ps, refs):
    a = torch.cat([p.detach().double().cpu().reshape(-1) for p in ps])
    b = torch.cat([p.detach().double().cpu().reshape(-1) for p in refs])
    return float((a - b).norm() / b.norm())


def _model(sd, C):
    m = dsk.DeepSpeakerModel(512, C).cuda().train()
    m.load_state_dict(sd)
    return m


@pytest.mark.parametrize("opt_kind", ["fused", "torch"])
def test_step_at_world_size_one(cuda_dev, opt_kind):
    C, K, topk, N, T = 1211, 3, 5, 64, 32
    sd = O.make_state_dict(0, num_classes=C)
    W0 = torch.randn(C * K, 512, generator=torch.Generator().manual_seed(9)).cuda() / 512 ** 0.5
    x = O.make_input(N, T, seed=5, scale=3.0).cuda()
    labels = torch.randint(0, C, (N,), generator=torch.Generator().manual_seed(5))
    # a unit initial accumulator keeps the first Adagrad update linear in the gradient (not its sign)
    make = (lambda ps: dsk.FusedAdagrad(ps, lr=1e-2, lr_decay=1e-4, initial_accumulator_value=1.0)) \
        if opt_kind == "fused" else \
        (lambda ps: torch.optim.Adagrad(ps, lr=1e-2, lr_decay=1e-4, initial_accumulator_value=1.0))
    ref_model = _model(sd, C)
    Wref = torch.nn.Parameter(W0.clone())
    ref_opt = make(list(ref_model.parameters()) + [Wref])
    ref = dsk.aam_softmax_step(ref_model, ref_opt, x, labels, margin=M, scale=SC, weight=Wref, subcentres=K, topk=topk,
                               topk_margin=TM)
    model = _model(sd, C)
    head = dsk.ShardedAAMSoftmaxLoss(W0, M, SC, subcentres=K, topk=topk, topk_margin=TM)
    opt, hopt = make(list(model.parameters())), make([head.weight])
    with pytest.raises(ValueError):
        dsk.sharded_aam_softmax_step(model, torch.optim.SGD(list(model.parameters()) + [head.weight], lr=0.0), x,
                                     labels, head=head, head_optimizer=hopt)
    out = dsk.sharded_aam_softmax_step(model, opt, x, labels, head=head, head_optimizer=hopt)
    assert abs(out["loss"].item() - ref["loss"].item()) <= 1e-5 * ref["loss"].item()
    dW = float((head.weight.detach() - Wref.detach()).abs().max() / (Wref.detach() - W0).abs().max())
    assert dW <= 1e-5, dW
    # the network against the reference step: rel-L2 over all its parameters (a parameter whose gradient is a
    # cancelling sum, such as a BatchNorm shift, differs more on its own: gE differs from the whole op's by ~1e-6)
    worst = _flat_rel(model.parameters(), ref_model.parameters())
    assert worst <= 1e-5, worst
    smodel = _model(sd, C).sync_batchnorm()
    shead = dsk.ShardedAAMSoftmaxLoss(W0, M, SC, subcentres=K, topk=topk, topk_margin=TM)
    sout = dsk.sharded_aam_softmax_step(smodel, make(list(smodel.parameters())), x, labels, head=shead,
                                        head_optimizer=make([shead.weight]))
    assert abs(sout["loss"].item() - ref["loss"].item()) <= 1e-3
    print(f"\n{opt_kind}: loss {out['loss'].item():.6f} vs {ref['loss'].item():.6f}, W {dW:.1e}, net {worst:.1e}")


# ---- NCCL ------------------------------------------------------------------------------------------------------------
N_LOCAL, T_STEP, C_STEP, K_STEP, TOPK_STEP = 16, 32, 1211, 3, 5


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _global_batch(world):
    N = world * N_LOCAL
    return O.make_input(N, T_STEP, seed=11, scale=3.0), torch.randint(0, C_STEP, (N,),
                                                                       generator=torch.Generator().manual_seed(11))


def _w0():
    return torch.randn(C_STEP * K_STEP, 512, generator=torch.Generator().manual_seed(3)) / 512 ** 0.5


def _nccl_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        sd = O.make_state_dict(0, num_classes=C_STEP)
        model = _model(sd, C_STEP).sync_batchnorm()
        head = dsk.ShardedAAMSoftmaxLoss(_w0().cuda(), M, SC, subcentres=K_STEP, topk=TOPK_STEP, topk_margin=TM,
                                         process_group=dist.group.WORLD)
        opt = dsk.FusedAdagrad(list(model.parameters()), lr=1e-2, lr_decay=1e-4, initial_accumulator_value=1.0)
        hopt = dsk.FusedAdagrad([head.weight], lr=1e-2, lr_decay=1e-4, initial_accumulator_value=1.0,
                                process_group=dist.group.WORLD)
        x, labels = _global_batch(world)
        res = dsk.sharded_aam_softmax_step(model, opt, P.shard(x, rank, world).cuda(), P.shard(labels, rank, world),
                                           head=head, head_optimizer=hopt)
        full = head.full_weight()
        torch.cuda.synchronize()
        out[rank] = dict(loss=res["loss"].cpu(), W=head.weight.detach().cpu(), rng=head.class_range, full=full.cpu(),
                         params=[p.detach().cpu().clone() for p in model.parameters()])
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_step_on_nccl(cuda_dev, world):
    visible = torch.cuda.device_count()
    if visible < world:
        pytest.skip(f"needs {world} GPUs, {visible} visible")
    port = _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_nccl_worker, args=(world, port, out), nprocs=world, join=True)
    res = [out[r] for r in range(world)]
    x, labels = _global_batch(world)
    model = _model(O.make_state_dict(0, num_classes=C_STEP), C_STEP).sync_batchnorm()
    W = torch.nn.Parameter(_w0().cuda())
    opt = dsk.FusedAdagrad(list(model.parameters()) + [W], lr=1e-2, lr_decay=1e-4, initial_accumulator_value=1.0)
    ref = dsk.aam_softmax_step(model, opt, x.cuda(), labels, margin=M, scale=SC, weight=W, subcentres=K_STEP,
                               topk=TOPK_STEP, topk_margin=TM)
    assert all(torch.equal(r["loss"], res[0]["loss"]) for r in res)
    assert abs(res[0]["loss"].item() - ref["loss"].item()) <= 1e-5 * ref["loss"].item()
    Wc = W.detach().cpu()
    for r in res:
        c0, c1 = r["rng"]
        assert float((r["W"] - Wc[c0 * K_STEP:c1 * K_STEP]).abs().max()) <= 1e-5
        assert torch.equal(r["full"], res[0]["full"])
    worst = _flat_rel(res[0]["params"], [p.detach().cpu() for p in model.parameters()])
    print(f"\nR={world}: loss {res[0]['loss'].item():.6f} vs {ref['loss'].item():.6f}, network rel-L2 {worst:.2e}")
    assert worst <= 1e-5
