"""DeepSpeakerModel.forward on the H100 engine vs the oracle and the reference's golden embeddings."""
import os

import numpy as np
import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from oracle import rescnn_oracle as O
from tests.helpers import rel_l2

pytestmark = pytest.mark.gpu

TOL = {"fp16": 1e-3, "bf16": 6e-3}   # north star: 1e-3 relative fp32 (met with fp16 operands; bf16 documented at ~3e-3)


@pytest.fixture(scope="module")
def models(cuda_dev):
    sd = O.make_state_dict(0, 16)
    out = {}
    for dt in ("fp16", "bf16"):
        m = dsk.DeepSpeakerModel(512, 16, operand_dtype=dt).to(cuda_dev).eval()
        m.load_state_dict(sd)
        out[dt] = m
    return sd, out


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
def test_eval_forward_matches_reference_golden(models, golden_dir, dt):
    sd, ms = models
    g = np.load(os.path.join(golden_dir, "eval_forward.npz"))
    for name in ("a", "b", "c"):
        B, T, seed, scale = g[f"{name}_cfg"]
        x = O.make_input(int(B), int(T), int(seed), float(scale)).cuda()
        with torch.no_grad():
            e = ms[dt](x)
        ref = torch.from_numpy(g[f"{name}_emb"])
        rel = ((e.cpu() - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
        assert rel < TOL[dt], (name, rel)
        assert torch.allclose(e.norm(dim=1).cpu(), torch.full((int(B),), 10.0), atol=1e-3)
        assert ms[dt].features is e          # side-effect attribute, model.py:210,213


@pytest.mark.parametrize("B,T", [(1, 160), (7, 160), (16, 48), (33, 32), (64, 160)])
def test_eval_forward_matches_oracle(models, B, T):
    sd, ms = models
    x = O.make_input(B, T, seed=100 + B, scale=5.0)
    with torch.no_grad():
        ref = O.forward(sd, x)
        e = ms["fp16"](x.cuda()).cpu()
    rel = ((e - ref).norm(dim=1) / ref.norm(dim=1))
    assert rel.max().item() < 1e-3
    # per-component gate: absolute error below 0.3 % of the RMS component (10/sqrt(512) = 0.44); the
    # floor-relative maximum of SURVEY §8d is a reported figure, not a gate (a near-zero component inflates it)
    assert (e - ref).abs().max().item() < 3e-3 * 10 / 512 ** 0.5


def test_full_size_properties(models):
    """BASELINE configs[1] size: determinism, unit-10 norms, batch-composition invariance (eval BN)."""
    sd, ms = models
    m = ms["fp16"]
    x = O.make_input(64, 160, seed=7, scale=8.0).cuda()
    with torch.no_grad():
        e1 = m(x).clone()
        e2 = m(x).clone()
        assert torch.equal(e1, e2)                                    # idempotent / deterministic
        assert torch.allclose(e1.norm(dim=1), torch.full((64,), 10.0, device=x.device), atol=1e-3)
        perm = torch.randperm(64, device=x.device)
        ep = m(x[perm].contiguous())
        # each utterance is independent of its batch (eval BN), bit for bit
        assert torch.equal(ep, e1[perm])
        e_small = m(x[5:8].contiguous())
        assert torch.equal(e_small, e1[5:8])
        assert torch.isfinite(m(torch.full_like(x, 1e4))).all()       # clip at 20 keeps everything finite


def test_weights_follow_parameter_updates(models):
    sd, ms = models
    m = dsk.DeepSpeakerModel(512, 16).cuda().eval()
    m.load_state_dict(sd)
    x = O.make_input(2, 32, seed=3).cuda()
    with torch.no_grad():
        e0 = m(x).clone()
        m.model.layer2[0].conv1.weight.mul_(1.5)          # in-place update bumps ._version -> repack
        sd2 = {k: v.clone() for k, v in sd.items()}
        sd2["model.layer2.0.conv1.weight"] = sd2["model.layer2.0.conv1.weight"] * 1.5
        e1 = m(x).cpu()
        ref = O.forward(sd2, x.cpu())
    assert rel_l2(e1, ref) < 1e-3 and rel_l2(e0.cpu(), ref) > 1e-3


def test_rejects_bad_input(models):
    sd, ms = models
    m = ms["fp16"]
    with pytest.raises(RuntimeError):
        m(torch.zeros(2, 1, 64, 160, device="cuda"))       # transposed layout (SURVEY §0 fact 1)
    with pytest.raises(RuntimeError, match="multiple of 16"):
        m(torch.zeros(2, 1, 100, 64, device="cuda"))


def _fresh_model(sd, env, dt="fp16"):
    """A model whose engine handle is created under the given environment knobs (read once by dsk_create)."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        m = dsk.DeepSpeakerModel(512, 16, operand_dtype=dt).cuda().eval()
        m.load_state_dict(sd)
        with torch.no_grad():
            m(O.make_input(1, 16, seed=1, scale=1.0).cuda())   # creates the handle now
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return m


def test_graph_launch_equals_kernel_by_kernel(models):
    """From the second call of a shape on, a forward is one CUDA-graph launch whose first / last kernel nodes are
    re-pointed at the call's input / output; it must be bit-identical to the 15 plain launches (DSK_GRAPH=0)."""
    sd, _ = models
    mg = _fresh_model(sd, {"DSK_GRAPH": "1"})
    mp = _fresh_model(sd, {"DSK_GRAPH": "0"})
    side = torch.cuda.Stream()      # the legacy default stream cannot be captured: the graph path needs a real stream
    cur = torch.cuda.current_stream()

    def graph_forward(x):
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            out = mg(x)
        cur.wait_stream(side)
        return out

    with torch.no_grad():
        for i in range(4):                      # call 0 plain (warm-up), call 1 captures, calls 2-3 re-target
            x = O.make_input(5, 48, seed=40 + i, scale=4.0).cuda()
            a = graph_forward(x)
            b = mp(x)
            assert torch.equal(a, b), i
        x = O.make_input(3, 32, seed=50, scale=4.0).cuda()   # a new shape drops the plan and its graph
        assert torch.equal(graph_forward(x), mp(x))
        x = O.make_input(5, 48, seed=51, scale=4.0).cuda()
        assert torch.equal(graph_forward(x), mp(x))


def test_graph_follows_weight_reload(models):
    sd, _ = models
    mm = _fresh_model(sd, {"DSK_GRAPH": "1"})
    side, cur = torch.cuda.Stream(), torch.cuda.current_stream()

    def m(x):                                   # on a capturable stream (see test_graph_launch_equals_kernel_by_kernel)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            out = mm(x)
        cur.wait_stream(side)
        return out

    x = O.make_input(4, 32, seed=60, scale=3.0).cuda()
    with torch.no_grad():
        for _ in range(3):
            e0 = m(x)
        mm.model.fc.bias.add_(0.25)             # bumps the parameter version -> weights reloaded, plans rebuilt
        cur.synchronize()
        e1 = m(x)
        e2 = m(x)
        ref = O.forward({k: v.cpu() for k, v in mm.state_dict().items()}, x.cpu())
    assert not torch.equal(e0, e1)
    assert torch.equal(e1, e2)
    assert ((e1.cpu() - ref).norm(dim=1) / ref.norm(dim=1)).max().item() < 1e-3
