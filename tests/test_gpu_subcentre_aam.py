"""Sub-centre AAM-softmax with the inter-top-k penalty on the GPU: the K = 1, topk = 0 call against the plain op bit for
bit, the class cosines, sub-centre argmax, top-k selection and loss against the fp64 oracle, the backward against the
oracle with the engine's cos / sub / top pinned, the branch cases, determinism and the batch split, non-finite inputs,
argument rejection, the sub-centre cosines and the training step end to end."""
import copy
import math
import zlib

import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import engine as EN
from deepspeaker_pytorch_b200 import frontend as FE
from oracle import rescnn_oracle as O
from oracle import subcentre_aam_oracle as S
from tests.test_gpu_aam_softmax import SHAPES, _row_rel

pytestmark = pytest.mark.gpu

M, SC, TM = 0.2, 30.0, 0.1


def _case(N, C, K, D, norms="norm10"):
    g = torch.Generator().manual_seed(zlib.crc32(f"sc{N}x{C}x{K}x{D}{norms}".encode()))
    E = torch.randn(N, D, generator=g)
    if norms == "norm10":
        E = 10.0 * E / E.norm(dim=1, keepdim=True)
    else:
        E = E * torch.exp(torch.empty(N, 1).uniform_(-4.0, 5.0, generator=g))
    W = torch.randn(C * K, D, generator=g) * (1.0 / D ** 0.5)
    return E, W, torch.randint(0, C, (N,), generator=g)


def _fwd(E, W, y, K, topk, m=M, s=SC, tm=TM):
    _, _, _, loss, cos, lse, sub, top = EN.aam_softmax_sc(E.cuda(), W.cuda(), y.cuda(), m, s, K, topk, tm)
    return loss.reshape(()), cos, lse, sub, top


def _bwd(E, W, y, cos, lse, sub, top, K, topk, m=M, s=SC, tm=TM, g=1.0):
    gl = torch.full((), float(g), device="cuda")
    return EN.aam_softmax_sc_backward(E.cuda().contiguous(), W.cuda().contiguous(), y.cuda(), cos, lse, sub, top, m, s,
                                      K, topk, tm, gl)


def _plain(E, W, y, m, s, g=1.0):
    """dsk_aam_softmax / dsk_aam_softmax_bwd called directly through the C ABI."""
    lib = L.load()
    E, W, y = E.cuda().contiguous(), W.cuda().contiguous(), y.cuda()
    (N, D), C = E.shape, W.shape[0]
    h = EN._allpairs_handle(E.device)
    loss, cos, lse = (torch.empty(1, device="cuda"), torch.empty(N, C, device="cuda"), torch.empty(N, device="cuda"))
    L.check(lib.dsk_aam_softmax(h, E.data_ptr(), W.data_ptr(), y.data_ptr(), N, C, D, m, s, loss.data_ptr(),
                                cos.data_ptr(), lse.data_ptr(), L.cur_stream()))
    gl = torch.full((1,), float(g), device="cuda")
    gE, gW = torch.empty_like(E), torch.empty_like(W)
    L.check(lib.dsk_aam_softmax_bwd(h, E.data_ptr(), W.data_ptr(), y.data_ptr(), cos.data_ptr(), lse.data_ptr(), N, C, D,
                                    m, s, gl.data_ptr(), gE.data_ptr(), gW.data_ptr(), L.cur_stream()))
    return loss.reshape(()), cos, lse, gE, gW


def _eq(a, b):
    return (a is None and b is None) or torch.equal(a, b)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_k1_topk0_is_the_plain_op_bit_for_bit(cuda_dev, shape):
    N, C, D = shape
    E, W, y = _case(N, C, 1, D, "arbitrary")
    for m, s in ((0.0, 30.0), (0.2, 30.0), (0.5, 64.0)):
        ref = _plain(E, W, y, m, s)
        loss, cos, lse, sub, top = _fwd(E, W, y, 1, 0, m, s, 0.0)
        gE, gW = _bwd(E, W, y, cos, lse, sub, top, 1, 0, m, s, 0.0)
        assert sub is None and top is None
        for a, b in zip((loss, cos, lse, gE, gW), ref):
            assert torch.equal(a, b), (m, s)


@pytest.mark.parametrize("K", [1, 3])
def test_topk_with_zero_margin_is_topk0_bit_for_bit(cuda_dev, K):
    E, W, y = _case(384, 1211, K, 512)
    ref = _fwd(E, W, y, K, 0, tm=0.0)
    ref_g = _bwd(E, W, y, *ref[1:], K, 0, tm=0.0)
    for topk in (5, 64):
        out = _fwd(E, W, y, K, topk, tm=0.0)
        for a, b in zip(out[:4], ref[:4]):
            assert _eq(a, b), topk
        for a, b in zip(_bwd(E, W, y, *out[1:], K, topk, tm=0.0), ref_g):
            assert torch.equal(a, b), topk


def _oracle_g(E, W):
    e = E.double() / E.double().norm(dim=1, keepdim=True).clamp_min(1e-12)
    w = W.double() / W.double().norm(dim=1, keepdim=True).clamp_min(1e-12)
    return e @ w.T


FWD_CASES = [(s, K) for s in ((384, 1211, 512), (1024, 5994, 512), (7, 3, 64)) for K in (2, 3, 5)] + \
    [((256, 3 * 5994, 512), 3)]


@pytest.mark.parametrize("shape,K", FWD_CASES, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else f"K{v}")
def test_forward_and_backward_vs_fp64(cuda_dev, shape, K):
    N, C, D = shape
    E, W, y = _case(N, C, K, D)
    g = _oracle_g(E, W)
    ref_cos, ref_sub = S.subcentre_max(g, K)
    top2 = g.reshape(N, C, K).topk(2, dim=2).values
    clear = (top2[..., 0] - top2[..., 1]) > 4e-6                 # the argmax is resolved by fp32 cosines
    cases = [t for t in (0, 5, 64) if t <= C - 1]
    for topk in cases:
        loss, cos, lse, sub, top = _fwd(E, W, y, K, topk)
        oloss, _, _, _, _ = S.forward(E, W, y, K, M, SC, topk, TM, cos=ref_cos, sub=ref_sub)
        dcos = float((cos.double().cpu() - ref_cos).abs().max())
        assert dcos <= 1e-6, (topk, dcos)
        assert abs(loss.item() - float(oloss)) <= 1e-5 * max(float(oloss), 1.0), (topk, loss.item(), float(oloss))
        subc = sub.cpu().to(torch.int64)
        assert torch.equal(subc[clear], ref_sub[clear]), topk
        if topk:
            assert torch.equal(top.cpu().to(torch.int64), S.select_topk(cos.cpu(), y, topk)), topk
        if topk == cases[-1]:                                      # the backward at the largest topk, cos/sub/top pinned
            gE, gW = _bwd(E, W, y, cos, lse, sub, top, K, topk)
            rE, rW = S.backward(E, W, y, K, M, SC, topk, TM, cos=cos.cpu(), sub=subc,
                                top=None if top is None else top.cpu().to(torch.int64))
            eE, eW = _row_rel(gE, rE), _row_rel(gW, rW)
            assert eE <= 1e-5 and eW <= 1e-5, (topk, eE, eW)
            chosen = torch.zeros(C * K, dtype=torch.bool)
            chosen[(torch.arange(C)[None, :] * K + subc).reshape(-1)] = True
            assert not bool(gW.cpu()[~chosen].any())
            print(f"\n{shape} K {K} topk {topk}: |dcos| {dcos:.2e}, gE {eE:.2e} gW {eW:.2e}, "
                  f"{int((~chosen).sum())} unchosen sub-centres")


def _branch_case(K=3):
    """Rows 0-7 past pi - m (all sub-centres of their class near the negated row); row 8 on sub-centre 1 of its class
    (sin = 0, cos = 1 exactly: a basis direction normalises without rounding); row 9 at cos = 1 with sub-centre 2 of a
    non-target class; class 42 with three equal sub-centres; class 43 with zero sub-centres."""
    N, C, D = 64, 100, 512
    E, W, y = _case(N, C, K, D)
    y = y.clone()
    y[:8] = torch.arange(8) + 50
    gn = torch.Generator().manual_seed(5)
    base = torch.randn(8, D, generator=gn) / D ** 0.5
    for k in range(K):
        W[y[:8] * K + k] = base + 0.01 * torch.randn(8, D, generator=gn) / D ** 0.5
    E[:8] = -10.0 * base / base.norm(dim=1, keepdim=True) + 0.02 * torch.randn(8, D, generator=gn)
    u, v = torch.zeros(D), torch.zeros(D)
    u[17], v[99] = 1.0, 1.0
    W[40 * K + 1], y[8], E[8] = 0.25 * u, 40, 10.0 * u
    W[41 * K + 2], y[9], E[9] = 0.25 * v, 7, 10.0 * v
    W[42 * K + 1] = W[42 * K + 2] = W[42 * K]
    y[10:12] = 42
    W[43 * K:44 * K] = 0.0
    y[12:14] = 43
    return E, W, y


@pytest.mark.parametrize("m,s,tm", [(0.0, 30.0, 0.0), (0.2, 30.0, 0.1), (0.5, 64.0, 0.3)])
def test_branch_cases(cuda_dev, m, s, tm):
    K, topk = 3, 5
    E, W, y = _branch_case(K)
    loss, cos, lse, sub, top = _fwd(E, W, y, K, topk, m, s, tm)
    c, sb, tp = cos.cpu(), sub.cpu().to(torch.int64), top.cpu().to(torch.int64)
    ref_cos, _ = S.subcentre_max(_oracle_g(E, W), K)
    assert float((c.double() - ref_cos).abs().max()) <= 1e-6
    oloss = S.forward(E, W, y, K, m, s, topk, tm, cos=ref_cos)[0]
    assert abs(loss.item() - float(oloss)) <= 1e-5 * max(float(oloss), 1.0)
    assert c[8, 40].item() == 1.0 and sb[8, 40] == 1
    assert c[9, 41].item() == 1.0 and sb[9, 41] == 2 and tp[9, 0] == 41
    assert not bool(sb[:, 42].any()) and not bool(c[:, 43].any()) and not bool(sb[:, 43].any())
    if m > 0:
        assert bool((c[torch.arange(8), y[:8]] < -math.cos(m)).all())
    gE, gW = _bwd(E, W, y, cos, lse, sub, top, K, topk, m, s, tm)
    assert bool(torch.isfinite(gE).all()) and bool(torch.isfinite(gW).all())
    rE, rW = S.backward(E, W, y, K, m, s, topk, tm, cos=c, sub=sb, top=tp)
    eE, eW = _row_rel(gE, rE), _row_rel(gW, rW)
    assert eE <= 1e-5 and eW <= 1e-5, (eE, eW)
    gW = gW.cpu()
    assert gW[43 * K].abs().sum().item() > 0 and not bool(gW[43 * K + 1:44 * K].any())
    assert not bool(gW[42 * K + 1:43 * K].any())


def test_deterministic(cuda_dev):
    K, topk = 3, 5
    E, W, y = _case(384, 1211, K, 512)
    runs = []
    for _ in range(2):
        out = _fwd(E, W, y, K, topk)
        runs.append(out + _bwd(E, W, y, *out[1:], K, topk))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("split", [(192, 192), (96, 96, 96, 96), (1, 127, 256)], ids=["R2", "R4", "uneven"])
def test_rows_do_not_depend_on_the_split(cuda_dev, split):
    K, topk = 3, 5
    E, W, y = _case(384, 1211, K, 512)
    N = E.shape[0]
    loss, cos, lse, sub, top = _fwd(E, W, y, K, topk)
    gE, _ = _bwd(E, W, y, cos, lse, sub, top, K, topk, g=N)
    _, gW = _bwd(E, W, y, cos, lse, sub, top, K, topk, g=1.0)
    gW_sum, lo = torch.zeros_like(gW, dtype=torch.float64), 0
    for n in split:
        sl = slice(lo, lo + n)
        _, c_r, l_r, s_r, t_r = _fwd(E[sl], W, y[sl], K, topk)
        assert torch.equal(c_r, cos[sl]) and torch.equal(l_r, lse[sl])
        assert torch.equal(s_r, sub[sl]) and torch.equal(t_r, top[sl])
        gE_r, _ = _bwd(E[sl], W, y[sl], c_r, l_r, s_r, t_r, K, topk, g=n)
        assert torch.equal(gE_r, gE[sl])
        _, gW_r = _bwd(E[sl], W, y[sl], c_r, l_r, s_r, t_r, K, topk, g=1.0)
        gW_sum += (n / N) * gW_r.double()
        lo += n
    rel = float((gW_sum - gW.double()).norm() / gW.double().norm())
    assert rel <= 1e-6, rel


def test_nan_embedding_row_is_contained(cuda_dev):
    K, topk = 3, 5
    E, W, y = _case(130, 1000, K, 192)
    clean = _fwd(E, W, y, K, topk)
    clean_g = _bwd(E, W, y, *clean[1:], K, topk)
    bad = E.clone()
    bad[17, 5] = float("nan")
    out = _fwd(bad, W, y, K, topk)
    g = _bwd(bad, W, y, *out[1:], K, topk)
    assert math.isnan(out[0].item())
    keep = torch.arange(130) != 17
    for a, b in zip(out[1:], clean[1:]):
        assert torch.equal(a[keep], b[keep])
    assert torch.equal(g[0][keep], clean_g[0][keep])
    t = out[4][17].cpu()
    assert bool(((t >= 0) & (t < 1000) & (t != y[17])).all())


def test_nan_subcentre_weight_row(cuda_dev):
    K, topk, C = 3, 5, 300
    E, W, y = _case(128, C, K, 192)
    W[7 * K + 1, 3] = float("nan")                       # class 7's sub-centre 1
    loss, cos, lse, sub, top = _fwd(E, W, y, K, topk)
    c, t = cos.cpu(), top.cpu().to(torch.int64)
    assert bool(torch.isnan(c[:, 7]).all()) and bool((sub.cpu()[:, 7] == 1).all())
    assert int(torch.isnan(c).sum()) == 128
    assert bool(((t >= 0) & (t < C) & (t != 7) & (t != y[:, None])).all())
    assert torch.equal(t, S.select_topk(c, y, topk))
    # fewer numbers than topk: the NaN class is selected last, never ahead of a number
    E2, W2, y2 = _case(8, 3, 2, 64)
    W2[1 * 2 + 0, 0] = float("nan")
    y2[:] = 0
    _, cos2, _, _, top2 = _fwd(E2, W2, y2, 2, 2)
    assert top2.cpu().tolist() == [[2, 1]] * 8 and bool(torch.isnan(cos2[:, 1]).all())


def test_bad_arguments_are_rejected(cuda_dev):
    E, y = torch.randn(8, 64, device="cuda"), torch.zeros(8, dtype=torch.long)
    for rows, kw in ((30, dict(subcentres=0)), (34, dict(subcentres=17)), (65538, dict(subcentres=2)),
                     (31, dict(subcentres=3)), (30, dict(subcentres=3, topk=10)), (200, dict(topk=65)),
                     (30, dict(topk_margin=-0.1)), (30, dict(topk_margin=math.nan)), (30, dict(topk_margin=math.inf))):
        with pytest.raises((ValueError, RuntimeError)):
            dsk.AAMSoftmaxLoss(torch.randn(rows, 64, device="cuda"), 0.2, 30.0, **kw).forward(E, y)
        with pytest.raises((ValueError, RuntimeError)):
            EN.aam_softmax_sc(E, torch.randn(rows, 64, device="cuda"), y, 0.2, 30.0, kw.get("subcentres", 1),
                              kw.get("topk", 0), kw.get("topk_margin", 0.0))


def test_subcentre_cosines(cuda_dev):
    K = 3
    E, W, y = _case(1024, 5994, K, 512, "arbitrary")
    sc = EN.subcentre_cosines(E.cuda(), W.cuda(), y.cuda(), K).cpu()
    e = E.double() / E.double().norm(dim=1, keepdim=True)
    w = (W.double() / W.double().norm(dim=1, keepdim=True)).reshape(-1, K, 512)[y]
    ref = torch.einsum("nd,nkd->nk", e, w)
    ulp = (torch.nextafter(ref.float(), torch.tensor(math.inf)) - ref.float()).double()
    assert bool(((sc.double() - ref).abs() <= ulp).all())
    _, cos, _, sub, _ = _fwd(E, W, y, K, 5)
    ar = torch.arange(1024)
    assert torch.equal(cos.cpu()[ar, y], sc.max(1).values)
    top2 = sc.topk(2, dim=1).values
    clear = top2[:, 0] > top2[:, 1]
    assert torch.equal(sub.cpu()[ar, y].to(torch.int64)[clear], sc.argmax(1)[clear])
    bad = y.clone()
    bad[3] = 5994
    assert bool(torch.isnan(EN.subcentre_cosines(E.cuda(), W.cuda(), bad.cuda(), K)[3]).all())


@pytest.mark.parametrize("opt_kind", ["fused", "torch"])
@pytest.mark.parametrize("N,T", [(64, 32), (384, 160)])
def test_subcentre_step_end_to_end(cuda_dev, N, T, opt_kind):
    C, K, topk, m, s, tm = 1211, 3, 5, 0.2, 30.0, 0.1
    sd = O.make_state_dict(0, num_classes=C)
    model = dsk.DeepSpeakerModel(512, C).cuda().train()
    model.load_state_dict(sd)
    ref_model = copy.deepcopy(model)
    Wsc = torch.nn.Parameter(torch.randn(C * K, 512, generator=torch.Generator().manual_seed(9)).cuda() / 512 ** 0.5)
    W0 = Wsc.detach().clone()
    params = list(model.parameters()) + [Wsc]
    opt = dsk.FusedAdagrad(params, lr=1e-3, lr_decay=1e-4) if opt_kind == "fused" else \
        torch.optim.Adagrad(params, lr=1e-3, lr_decay=1e-4)
    x = O.make_input(N, T, seed=N, scale=3.0)
    labels = torch.randint(0, C, (N,), generator=torch.Generator().manual_seed(N))
    cls0 = {k: v.detach().clone() for k, v in model.model.classifier.named_parameters()}
    keys0 = list(model.state_dict().keys())
    seen = {}

    def hook(mod, inp, out):
        seen["emb"] = out.detach().clone()
        out.register_hook(lambda gr: seen.__setitem__("grad", gr.detach().clone()))

    h = model.register_forward_hook(hook)
    kw = dict(margin=m, scale=s, weight=Wsc, subcentres=K, topk=topk, topk_margin=tm)
    out = dsk.aam_softmax_step(model, opt, x.cuda(), labels, **kw)
    h.remove()
    assert out["loss"].dim() == 0 and out["loss"].is_cuda
    Ec, Wc, lab, loss, cos, lse, sub, top = EN.aam_softmax_sc(seen["emb"], W0, labels, m, s, K, topk, tm)
    gE, _ = EN.aam_softmax_sc_backward(Ec, Wc, lab, cos, lse, sub, top, m, s, K, topk, tm, torch.ones((), device="cuda"))
    assert torch.equal(seen["grad"], gE) and torch.equal(loss.reshape(()), out["loss"])
    with torch.no_grad():
        ref_emb = O.forward(sd, x, train=True)
    oloss = S.forward(ref_emb, W0.cpu(), labels, K, m, s, topk, tm)[0]
    assert abs(out["loss"].item() - float(oloss)) <= 1e-3, (out["loss"].item(), float(oloss))
    assert not torch.equal(Wsc.detach(), W0)
    for k, v in model.model.classifier.named_parameters():
        assert torch.equal(v.detach(), cls0[k]), k
    assert list(model.state_dict().keys()) == keys0
    with torch.no_grad():
        ref_model(x.cuda())
    for (k, v), (_, r) in zip(model.state_dict().items(), ref_model.state_dict().items()):
        if "running" in k:
            assert torch.equal(v, r), k
    sync_model = dsk.DeepSpeakerModel(512, C).cuda().train()
    sync_model.load_state_dict(sd)
    sync_model.sync_batchnorm()
    Ws2 = torch.nn.Parameter(W0.clone())
    sopt = dsk.FusedAdagrad(list(sync_model.parameters()) + [Ws2], lr=1e-3, lr_decay=1e-4)
    sout = dsk.aam_softmax_step(sync_model, sopt, x.cuda(), labels, **{**kw, "weight": Ws2})
    assert abs(sout["loss"].item() - out["loss"].item()) <= 1e-3
    print(f"\nN={N} T={T} {opt_kind}: loss {out['loss'].item():.6f} (oracle {float(oloss):.6f}, "
          f"sync BN {sout['loss'].item():.6f})")


def test_subcentre_step_on_speed_extended_labels(cuda_dev):
    C, K, N = 400, 3, 64
    plan = {"speeds": (0.9, 1.0, 1.1), "speed_idx": torch.arange(N) % 3}
    labels = FE.speed_labels(torch.arange(N) % C, plan, C)
    assert int(labels.max()) >= 2 * C
    model = dsk.DeepSpeakerModel(512, 3 * C).cuda()
    model.load_state_dict(O.make_state_dict(0, num_classes=3 * C))
    model.train()
    W = torch.nn.Parameter(torch.randn(3 * C * K, 512, device="cuda") / 512 ** 0.5)
    opt = dsk.FusedAdagrad(list(model.parameters()) + [W], lr=1e-2, lr_decay=1e-4)
    x = O.make_input(N, 32, seed=3, scale=3.0).cuda()
    out = dsk.aam_softmax_step(model, opt, x, labels, margin=0.2, scale=30.0, weight=W, subcentres=K, topk=5,
                               topk_margin=0.1)
    assert torch.isfinite(out["loss"]).all()
