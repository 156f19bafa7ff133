"""Synchronised BatchNorm: R model copies loaded from one state dict are driven in lockstep in one process, each
with its shard of the batch, their per-utterance records concatenated in rank order at every stage (what the
all_gather of a process group delivers).  What each shard computes must be bit-identical to its rows of the
one-shard forward, the statistics must pass the fp64 layer-by-layer checker, and the backward summed over shards must
be the one-shard backward."""
import ctypes
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import train as TR
from deepspeaker_pytorch_b200.engine import conv_bn_modules
from oracle import rescnn_oracle as O
from tests.helpers import rel_l2
from tests.test_gpu_backward_ops import TD, U
from tests.test_gpu_layer_parity import check_train_chain, stat_chains

pytestmark = pytest.mark.gpu


def _model(sd, dt="fp16", sync=True):
    m = dsk.DeepSpeakerModel(512, 16, operand_dtype=dt).cuda()
    m.load_state_dict(sd)
    m.train()
    return m.sync_batchnorm() if sync else m


def _concat(local):
    g = torch.cat(local)
    return [g] * len(local)


def _running(m):
    return [t.detach().clone() for _, bn in conv_bn_modules(m) for t in (bn.running_mean, bn.running_var)]


def _read(m, tctx, B, T, which, layer):
    st = layer // 3
    t = torch.empty(B, 64 << st, T >> (st + 1), 64 >> (st + 1), device="cuda")
    eng = m._engine
    L.check(eng.lib.dsk_train_ctx_read(eng.handle, tctx, which, layer, t.data_ptr(), L.cur_stream()), "dsk_train_ctx_read")
    return t


def lockstep_forward(models, shards):
    """The synchronised forward of every shard on its own model copy, one exchange per stage for all of them."""
    engs, embs = [], []
    for m, x in zip(models, shards):
        eng = m._get_engine(x.device)
        eng.sync_weights(eval_mode=False)
        engs.append(eng)
        embs.append(torch.empty(x.shape[0], 512, device="cuda"))
    ctxs = TR.run_lockstep([TR.sync_forward_stages(e, x, o) for e, x, o in zip(engs, shards, embs)], _concat)
    return engs, embs, ctxs


def lockstep_backward(models, engs, ctxs, grad_embs):
    """The staged backward of each copy into fresh gradient tensors (38 per copy)."""
    views, gens = [], []
    for m, e, c, ge in zip(models, engs, ctxs, grad_embs):
        v = [torch.empty_like(p) for p in TR._train_params(m)]
        views.append(v)
        gens.append(TR.sync_backward_stages(e, c, ge.shape[0], ge.contiguous(), v))
    TR.run_lockstep(gens, _concat)
    torch.cuda.synchronize()
    return views


def _release(models, ctxs):
    for m, c in zip(models, ctxs):
        L.check(m._engine.lib.dsk_train_ctx_release(m._engine.handle, c), "dsk_train_ctx_release")


# ---- 1. split invariance of the forward ------------------------------------------------------------------------------
SPLIT_CASES = [(64, 32, (1, 2, 4, 8)), (384, 160, (1, 2, 4, 8)), (8, 32, (8,))]


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
@pytest.mark.parametrize("N,T,Rs", SPLIT_CASES, ids=[f"N{n}_T{t}" for n, t, _ in SPLIT_CASES])
def test_forward_is_split_invariant(cuda_dev, dt, N, T, Rs):
    sd = O.make_state_dict(11, 16)
    x = O.make_input(N, T, 900 + N, 3.0).cuda()
    m1 = [_model(sd, dt)]
    _, (e1,), (c1,) = lockstep_forward(m1, [x])
    run1 = _running(m1[0])
    for R in Rs:
        n = N // R
        ms = [_model(sd, dt) for _ in range(R)]
        engs, embs, ctxs = lockstep_forward(ms, [x[r * n:(r + 1) * n] for r in range(R)])
        torch.cuda.synchronize()
        assert torch.equal(torch.cat(embs), e1), f"R={R}: embeddings differ"
        for i in range(12):
            for which in (0, 1):
                ref = _read(m1[0], c1, N, T, which, i)
                got = torch.cat([_read(m, c, n, T, which, i) for m, c in zip(ms, ctxs)])
                assert torch.equal(got, ref), f"R={R}: {'y' if which else 'raw'}[{i}] differs from the one-shard forward"
                del ref, got
        for m in ms:
            assert all(torch.equal(a, b) for a, b in zip(_running(m), run1)), f"R={R}: running statistics differ"
        _release(ms, ctxs)
    _release(m1, [c1])


# ---- 2. accuracy ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt,B,T", [("fp16", 128, 160), ("bf16", 16, 48)])
def test_one_shard_forward_passes_the_layer_checker(cuda_dev, dt, B, T):
    sd = O.make_state_dict(6, 16)
    m = _model(sd, dt)
    x = O.make_input(B, T, 400 + B, 3.0).cuda()
    rm0 = [bn.running_mean.detach().clone() for _, bn in conv_bn_modules(m)]
    rv0 = [bn.running_var.detach().clone() for _, bn in conv_bn_modules(m)]
    emb = m(x)
    tctx = emb.grad_fn.guards[0].tctx
    raw = {i: _read(m, tctx, B, T, 0, i) for i in range(12)}
    y = {i: _read(m, tctx, B, T, 1, i) for i in range(12)}
    torch.cuda.synchronize()
    rm1 = [bn.running_mean.detach().clone() for _, bn in conv_bn_modules(m)]
    rv1 = [bn.running_var.detach().clone() for _, bn in conv_bn_modules(m)]
    chains = stat_chains(m._engine, tctx, B, T, sync=True)
    check_train_chain(f"sync {dt} B={B} T={T}", sd, dt, x, raw, y, emb, rm0, rv0, rm1, rv1, chains)


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
@pytest.mark.parametrize("C,B,HW", [(64, 128, 80 * 32), (512, 128, 10 * 4)])
@pytest.mark.parametrize("offset", [0, 1000])
def test_record_statistics_building_block(cuda_dev, dt, C, B, HW, offset):
    """y within 2u of the fp64 BatchNorm at channel mean/std up to 1000 (the bar of dsk_bn_act_train_forward)."""
    lib = L.load()
    h = ctypes.c_void_p()
    L.check(lib.dsk_create(ctypes.byref(h), 0, L.DSK_BF16 if dt == "bf16" else L.DSK_F16), "dsk_create")
    try:
        g = torch.Generator().manual_seed(C + offset)
        M = B * HW
        raw = torch.randn(M, C, generator=g) * 3.0 + torch.randn(C, generator=g)
        if offset:
            raw = torch.randn(M, C, generator=g) + torch.logspace(0, float(np.log10(offset)), C)[torch.randperm(C, generator=g)]
        gamma = torch.empty(C).uniform_(0.5, 1.5, generator=g)
        beta = torch.randn(C, generator=g) * 0.5 + 1.0
        rm, rv = torch.randn(C, generator=g) * 0.1, torch.empty(C).uniform_(0.5, 1.5, generator=g)
        res = (torch.randn(M, C, generator=g) * 2).to(TD[dt])
        rmr, rvr = rm.double().clone(), rv.double().clone()
        pre = torch.nn.functional.batch_norm(raw.double(), rmr, rvr, gamma.double(), beta.double(), True, 0.1, 1e-5)
        yr = (pre + res.double()).clamp(0, 20)
        d = lambda t: t.cuda().contiguous()
        rawd, gd, bd, rmd, rvd, resd = d(raw), d(gamma), d(beta), d(rm), d(rv), d(res)
        y16 = torch.empty(M, C, dtype=TD[dt], device="cuda")
        mean, rstd = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
        L.check(lib.dsk_bn_act_sync_train_forward(h, rawd.data_ptr(), gd.data_ptr(), bd.data_ptr(), rmd.data_ptr(),
                                                  rvd.data_ptr(), resd.data_ptr(), y16.data_ptr(), mean.data_ptr(),
                                                  rstd.data_ptr(), B, HW, C, L.cur_stream()), "bn sync fwd")
        torch.cuda.synchronize()
        assert torch.allclose(y16.float().cpu().double(), yr, rtol=2 * U[dt], atol=2e-3)
        assert torch.allclose(rmd.cpu().double(), rmr, rtol=1e-5, atol=1e-6)
        assert torch.allclose(rvd.cpu().double(), rvr, rtol=1e-5, atol=1e-6)
        assert torch.allclose(mean.cpu().double(), raw.double().mean(0), rtol=1e-5, atol=1e-5)
    finally:
        lib.dsk_destroy(h)


# ---- 3. against the oracle, and that it matters ----------------------------------------------------------------------
def test_two_shards_match_the_oracle_over_the_whole_batch(cuda_dev):
    sd = O.make_state_dict(3, 16)
    n, T = 16, 64
    x = torch.cat([O.make_input(n, T, 31, 1.0), O.make_input(n, T, 32, 3.0)])
    ref = O.forward(sd, x, True, {})
    rel = lambda e: rel_l2(e.cpu().double(), ref.double())
    xs = [x[:n].cuda(), x[n:].cuda()]
    ms = [_model(sd) for _ in range(2)]
    _, embs, ctxs = lockstep_forward(ms, xs)
    torch.cuda.synchronize()
    err_sync = rel(torch.cat(embs))
    _release(ms, ctxs)
    per_replica = _model(sd, sync=False)
    with torch.no_grad():
        err_default = rel(torch.cat([per_replica(xi) for xi in xs]))
        err_one_device = rel(_model(sd, sync=False)(x.cuda()))     # the default path with the whole batch on one GPU
    print(f"\nR=2 vs the fp32 oracle over the whole batch, rel-L2: synchronised {err_sync:.3e}, "
          f"per-replica {err_default:.3e}; default path, whole batch on one device {err_one_device:.3e}")
    # the train-mode bar is 1e-3; where the one-device forward of this batch itself sits at it, the synchronised
    # shards must be as close to the oracle as that forward
    assert err_sync < max(1e-3, 1.05 * err_one_device)
    assert err_default > 10 * 1e-3


# ---- 4. backward -----------------------------------------------------------------------------------------------------
def _grad_embs(N, R, seed=7):
    """Rows whose magnitude differs by 2^12 between neighbouring shards (the ranks must agree on one loss scale)."""
    g = torch.randn(N, 512, generator=torch.Generator().manual_seed(seed))
    n = N // R if R > 1 else N // 2
    scale = torch.tensor([4096.0 if (i // n) % 2 else 1.0 for i in range(N)]).view(N, 1)
    return (g * scale * 1e-4).cuda()


def _sharded_backward(sd, x, ge, R):
    n = x.shape[0] // R
    ms = [_model(sd) for _ in range(R)]
    engs, _, ctxs = lockstep_forward(ms, [x[r * n:(r + 1) * n] for r in range(R)])
    views = lockstep_backward(ms, engs, ctxs, [ge[r * n:(r + 1) * n] for r in range(R)])
    out = []
    for k in range(38):                       # what the data-parallel reduction does: add the ranks' shares
        acc = views[0][k].clone()
        for v in views[1:]:
            acc += v[k]
        out.append(acc)
    return out


def test_backward_summed_over_shards_is_the_one_shard_backward(cuda_dev):
    sd = O.make_state_dict(5, 16)
    N, T = 64, 48
    x = O.make_input(N, T, 77, 3.0).cuda()
    ge = _grad_embs(N, 2)
    ref = _sharded_backward(sd, x, ge, 1)
    assert all(torch.isfinite(t).all() for t in ref)
    again = _sharded_backward(sd, x, ge, 1)
    assert all(torch.equal(a, b) for a, b in zip(ref, again)), "two runs differ"
    for R in (2, 4):
        got = _sharded_backward(sd, x, ge, R)
        worst, same = 0.0, 0
        for a, b in zip(got, ref):
            worst = max(worst, float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)))
            same += int(torch.equal(a, b))
        print(f"\nR={R}: summed gradients vs one shard: worst rel-L2 {worst:.3e}, bit-identical tensors {same}/38")
        assert worst <= 1e-5
        twice = _sharded_backward(sd, x, ge, R)
        assert all(torch.equal(a, b) for a, b in zip(got, twice)), f"R={R}: two runs differ"


# ---- 5. triplet forward and the training steps -----------------------------------------------------------------------
def test_forward_triplet_equals_three_sequential_calls(cuda_dev):
    sd = O.make_state_dict(8, 16)
    xs = [O.make_input(12, 48, 60 + k, 3.0).cuda() for k in range(3)]
    w = [torch.randn(12, 512, generator=torch.Generator().manual_seed(k)).cuda() for k in range(3)]
    m1, m2 = _model(sd), _model(sd)
    outs1 = m1.forward_triplet(*xs)
    sum((o * wk).sum() for o, wk in zip(outs1, w)).backward()
    outs2 = [m2(x) for x in xs]
    sum((o * wk).sum() for o, wk in zip(outs2, w)).backward()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs1, outs2))
    assert all(torch.equal(a, b) for a, b in zip(m1.state_dict().values(), m2.state_dict().values()))
    for (k, p1), p2 in zip(m1.named_parameters(), m2.parameters()):
        assert (p1.grad is None) == (p2.grad is None), k
        assert p1.grad is None or torch.equal(p1.grad, p2.grad), k


def test_steps_on_a_synchronised_model(cuda_dev):
    sd = O.make_state_dict(9, 16)
    m = _model(sd)
    opt = dsk.FusedAdagrad(m.parameters(), lr=1e-3)
    x = O.make_input(32, 48, 90, 3.0).cuda()
    labels = torch.arange(32) % 8
    r = dsk.batch_hard_step(m, opt, x, labels, margin=0.5)
    r2 = dsk.batch_hard_step(m, opt, x, labels, margin=0.5, across_ranks=True)
    assert torch.isfinite(r["loss"]) and torch.isfinite(r2["loss"])
    ref = _model(sd, sync=False)
    r_ref = dsk.batch_hard_step(ref, dsk.FusedAdagrad(ref.parameters(), lr=1e-3), x, labels, margin=0.5)
    assert abs(float(r["loss"]) - float(r_ref["loss"])) <= 1e-3 * abs(float(r_ref["loss"]))
    xa, xp, xn = (O.make_input(8, 48, 95 + k, 3.0).cuda() for k in range(3))
    lp, ln = torch.arange(8), torch.arange(8) + 8
    a = dsk.train_step(m, opt, xa, xp, xn, lp, ln, margin=0.1, epoch=5)
    assert torch.isfinite(a["loss"])
    before = _running(m)
    with pytest.raises(ValueError):
        dsk.train_step(m, opt, xa, xp, xn, lp, ln, margin=0.1, epoch=1)
    assert all(torch.equal(u, v) for u, v in zip(before, _running(m)))        # refused before any forward


def test_turning_it_off_restores_the_default_path(cuda_dev):
    sd = O.make_state_dict(10, 16)
    x = O.make_input(16, 48, 99, 3.0).cuda()
    m = _model(sd).sync_batchnorm(False)
    ref = _model(sd, sync=False)
    assert torch.equal(m(x), ref(x))
    assert all(torch.equal(a, b) for a, b in zip(_running(m), _running(ref)))


def test_out_of_sequence_calls_are_refused(cuda_dev):
    sd = O.make_state_dict(12, 16)
    m = _model(sd)
    eng = m._get_engine(torch.device("cuda:0"))
    eng.sync_weights(eval_mode=False)
    x = O.make_input(4, 32, 1, 3.0).cuda()
    emb = torch.empty(4, 512, device="cuda")
    lib, h, s = eng.lib, eng.handle, L.cur_stream()
    tctx = ctypes.c_void_p()
    L.check(lib.dsk_sync_forward_begin(h, x.data_ptr(), 4, 32, emb.data_ptr(), ctypes.byref(tctx), s), "begin")
    g = L.DskGrads()
    assert lib.dsk_sync_backward_begin(h, tctx, emb.data_ptr(), ctypes.byref(g), s) == -3   # forward not finished
    assert lib.dsk_train_ctx_read(h, tctx, 0, 0, emb.data_ptr(), s) == -3
    more = ctypes.c_int32()
    assert lib.dsk_sync_stage(h, tctx, emb.data_ptr(), 3, ctypes.byref(more), s) == -1      # fewer than B records
    L.check(lib.dsk_train_ctx_release(h, tctx), "release")
    assert lib.dsk_sync_stage(h, tctx, emb.data_ptr(), 4, ctypes.byref(more), s) == -3
    p, nb = ctypes.c_void_p(), ctypes.c_int64()
    assert lib.dsk_sync_records(h, tctx, ctypes.byref(p), ctypes.byref(nb)) == -3
    e2 = _model(sd, sync=False)                                                               # a plain forward's context
    out = e2(x)
    assert lib.dsk_sync_backward_begin(e2._engine.handle, out.grad_fn.guard.tctx, emb.data_ptr(), ctypes.byref(g), s) == -3


# ---- 7. NCCL ------------------------------------------------------------------------------------------------------------
N_LOCAL, T_NCCL = 16, 48


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _nccl_batch(world):
    N = world * N_LOCAL
    return O.make_input(N, T_NCCL, 123, 3.0), (torch.arange(N) % 8).long()


def _nccl_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from deepspeaker_pytorch_b200.parallel import shard

        m = dsk.DeepSpeakerModel(512, 16).cuda()
        m.load_state_dict(O.make_state_dict(0, 16))
        m.train()
        m.sync_batchnorm()
        opt = dsk.FusedAdagrad(m.parameters(), lr=1e-3, lr_decay=1e-4)
        x, labels = _nccl_batch(world)
        seen = {}
        hook = m.register_forward_hook(lambda mod, inp, o: seen.__setitem__("emb", o.detach().clone()))
        res = dsk.batch_hard_step(m, opt, shard(x, rank, world).cuda(), shard(labels, rank, world), margin=0.5,
                                  across_ranks=True)
        hook.remove()
        torch.cuda.synchronize()
        out[rank] = dict(loss=res["loss"].cpu(), emb=seen["emb"].cpu(), running=[t.cpu() for t in _running(m)])
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_synchronised_batch_hard_step_on_nccl(cuda_dev, world):
    visible = torch.cuda.device_count()
    if visible < world:
        pytest.skip(f"needs {world} GPUs, {visible} visible")
    port = _free_port()
    out = mp.Manager().dict()
    mp.spawn(_nccl_worker, args=(world, port, out), nprocs=world, join=True)
    res = [out[r] for r in range(world)]
    x, labels = _nccl_batch(world)
    m = _model(O.make_state_dict(0, 16))
    with torch.no_grad():
        emb = m(x.cuda())
    loss = dsk.BatchHardTripletLoss(0.5).forward(emb, labels.cuda())
    assert torch.equal(torch.cat([r["emb"] for r in res]), emb.cpu())
    assert all(torch.equal(r["loss"], loss.reshape(()).cpu()) for r in res)
    for r in res:
        assert all(torch.equal(a, b.cpu()) for a, b in zip(r["running"], _running(m)))
