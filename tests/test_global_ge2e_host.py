"""GlobalGE2ELoss, host side (CPU, gloo, world size 2): the engine's four GE2E row-range ops are replaced in each worker by
stand-ins built from the fp64 GE2E oracle (the whole-batch forward sliced to the rank's rows; the mean; the oracle's
score gradients sliced to the rank's rows; and the gradient of sum(dcos * cos) over the whole batch, differentiated by
autograd from the gathered dcos), so the plumbing is checked without a GPU: the rank offsets, the global speaker lists
and V, the loss over the union, the gathered dcos, the per-rank gradient rows, the w and b shares and the collectives
issued."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from deepspeaker_pytorch_b200.parallel import gather_labels
from oracle import ge2e_oracle as G

W, B = 10.0, -5.0
METHODS = ("softmax", "contrast")
COLLECTIVES = ("all_gather_into_tensor", "all_gather", "all_reduce", "broadcast", "reduce_scatter_tensor",
               "all_to_all_single", "barrier", "send", "recv")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _batch():
    g = torch.Generator().manual_seed(11)
    E = torch.randn(24, 16, generator=g)
    labels = torch.arange(24) % 5                 # speakers of 4 or 5 rows, every one on both shards
    E = E + 2.0 * torch.randn(5, 16, generator=g)[labels]
    labels[23] = 40                               # a singleton on rank 1: no loss term, but a centroid column
    return E, labels


def _dcos(col, cos, rec, w, b, method, grad_loss):
    """(dS, dcos) of the whole batch at the oracle's cosines (and contrast argmax)."""
    dS = G.score_grads(cos, col, w, b, method, grad_loss, argmax=rec if method == "contrast" else None)
    return dS, max(w, 1e-6) * dS


def _install_stand_ins(EN, log, stash):
    def rows(E, csr, V, w, b, method, row0, n):
        log["rows"].append((int(row0), int(n), E.shape[0]))
        _, offsets, col = csr
        loss, cos, rec = G.forward(E, col, float(w), float(b), method)
        S = max(float(w), 1e-6) * cos + float(b)
        ar = torch.arange(col.numel())
        sig = torch.sigmoid(S)
        row = rec - S[ar, col] if method == "softmax" else 1.0 - sig[ar, col] + sig[ar, rec]
        valid = (offsets[1:] - offsets[:-1])[col] >= 2
        stash.update(cos=cos, rec=rec, row_loss=row * valid, V=V)
        sl = slice(row0, row0 + n)
        return E, cos[sl].clone(), rec[sl].clone(), (row * valid)[sl].clone()

    def mean(row_loss, V):
        log["mean_in"] = row_loss.clone()
        return (row_loss.double().sum() / V).reshape(1)

    def dcos_rows(cos, rec, csr, V, w, b, method, row0, n, grad_loss):
        sl = slice(row0, row0 + n)
        log["dcos"].append((int(row0), int(n), torch.equal(cos, stash["cos"][sl]), torch.equal(rec, stash["rec"][sl])))
        _, _, col = csr
        dS, dcos = _dcos(col, stash["cos"], stash["rec"], float(w), float(b), method, float(grad_loss))
        ar = torch.arange(col.numel())
        tdc = dcos[ar, col]
        dcos[ar, col] = 0.0
        gw = (dS[sl] * stash["cos"][sl]).sum() if float(w) >= 1e-6 else torch.zeros((), dtype=torch.float64)
        gb = dS[sl].sum() if method == "contrast" else torch.zeros((), dtype=torch.float64)
        return dcos[sl].clone(), tdc[sl].clone(), gw, gb

    def backward_rows(E, csr, dcos, tdc, row0, n):
        log["bwd"] = (int(row0), int(n), dcos.clone(), tdc.clone())
        _, _, col = csr
        full = dcos.double().clone()
        full[torch.arange(col.numel()), col] = tdc.double()
        with torch.enable_grad():                  # autograd runs a Function's backward with grad mode off
            E64 = E.double().requires_grad_(True)
            _, cos, _ = G.forward(E64, col, W, B, "softmax")
            g, = torch.autograd.grad((cos * full).sum(), E64)
        return g[row0:row0 + n]

    EN.ge2e_rows = rows
    EN.ge2e_mean = mean
    EN.ge2e_dcos_rows = dcos_rows
    EN.ge2e_backward_rows = backward_rows


def _count_collectives(counter):
    for name in COLLECTIVES:
        fn = getattr(dist, name)

        def wrapped(*a, _fn=fn, _name=name, **k):
            counter.append(_name)
            return _fn(*a, **k)

        setattr(dist, name, wrapped)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import deepspeaker_pytorch_b200 as dsk
        from deepspeaker_pytorch_b200 import engine as EN

        calls = []
        _count_collectives(calls)
        E, labels = _batch()
        n = E.shape[0] // world
        glabels = gather_labels(labels[rank * n:(rank + 1) * n])
        res = {"glabels": glabels.clone(), "n_label_collectives": len(calls)}
        for method in METHODS:
            log, stash = {"rows": [], "dcos": []}, {}
            _install_stand_ins(EN, log, stash)
            crit = dsk.GE2ELoss(W, B, method).double()
            local = E[rank * n:(rank + 1) * n].double().requires_grad_(True)
            n0 = len(calls)
            loss = dsk.GlobalGE2ELoss(crit).forward(local, glabels)
            n1 = len(calls)
            loss.backward()
            res[method] = dict(loss=loss.detach().clone(), grad=local.grad.clone(), gw=crit.w.grad.clone(),
                               gb=crit.b.grad.clone(), rows=log["rows"], dcos=log["dcos"], bwd=log["bwd"],
                               mean_in=log["mean_in"], V=stash["V"], fwd_calls=calls[n0:n1], bwd_calls=calls[n1:])
        out[rank] = res
    finally:
        dist.destroy_process_group()


def test_global_ge2e_plumbing_against_the_oracle():
    world = 2
    port = _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    E, labels = _batch()
    N, n = E.shape[0], E.shape[0] // world
    col, P, counts = G.speakers(labels)
    ar = torch.arange(N)
    for method in METHODS:
        oloss, ocos, orec = G.forward(E, labels, W, B, method)
        gE, gw, gb = G.backward(E, labels, W, B, method, cos=ocos, argmax=orec if method == "contrast" else None)
        _, odcos = _dcos(col, ocos, orec, W, B, method, 1.0)
        otdc = odcos[ar, col].clone()
        odcos[ar, col] = 0.0
        for r in range(world):
            o, sl = out[r][method], slice(r * n, (r + 1) * n)
            assert o["V"] == N - 1                                                    # the singleton has no term
            assert o["rows"] == [(r * n, n, N)]                                       # this rank's rows, all N
            assert o["dcos"] == [(r * n, n, True, True)]                              # its own cos / rec rows
            assert torch.equal(o["mean_in"], out[0][method]["mean_in"])               # every rank's row losses
            assert o["fwd_calls"] == ["all_gather_into_tensor"] * 2
            assert o["bwd_calls"] == ["all_gather_into_tensor"]
            assert o["loss"].dim() == 0 and abs(float(o["loss"]) - float(oloss)) <= 1e-12 * float(oloss)
            row0, rows, dcos, tdc = o["bwd"]
            assert (row0, rows) == (r * n, n)
            assert torch.allclose(dcos, odcos, rtol=0, atol=1e-15) and torch.allclose(tdc, otdc, rtol=0, atol=1e-15)
            err = float((o["grad"] - gE[sl]).norm() / gE[sl].norm())
            assert err <= 1e-10, (method, r, err)
        assert torch.equal(out[0][method]["loss"], out[1][method]["loss"])
        sw = float(out[0][method]["gw"] + out[1][method]["gw"])
        sb = float(out[0][method]["gb"] + out[1][method]["gb"])
        assert abs(sw - gw) <= 1e-10 * abs(gw)
        if method == "softmax":
            assert sb == 0.0
        else:
            assert abs(sb - gb) <= 1e-10 * max(abs(gb), 1e-12)
    for r in range(world):
        assert torch.equal(out[r]["glabels"], labels) and out[r]["n_label_collectives"] == 1
