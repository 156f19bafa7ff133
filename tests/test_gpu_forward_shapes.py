"""The eval forward at the shapes production runs: batches of 256 and more, and long utterances.

- Batch invariance, bit for bit.  Each output element of each kernel sums its products in an order that does not
  depend on the batch, so an utterance's embedding and every activation of it must have the same bits in any batch,
  with the forward as one CUDA graph and launched kernel by kernel.
- Every layer against fp64 (test_gpu_layer_parity.py's checker) at the batch `embed_utterances` forwards, one past it,
  and a long utterance.
- Long utterances past the bound of the halo epilogue's old 32-bit reciprocal (test_halo_index_host.py computes the
  shapes), and the halo conv alone at a tall geometry past it.
"""
import ctypes
import gc

import pytest
import torch
import torch.nn.functional as F

from deepspeaker_pytorch_b200 import _lib as L
from oracle import rescnn_oracle as O
from tests.test_gpu_forward import _fresh_model
from tests.test_gpu_halo_conv import from_planar, hl, to_padded  # noqa: F401  (hl: the fixture)
from tests.test_gpu_layer_parity import eval_case, read_eval_activations, unpack_eval_activations
from tests.test_halo_index_host import GIB, OLD_FAILS, TALL_OP, eval_workspace, first_failing_batch

pytestmark = pytest.mark.gpu

POOL = 300
WHOLE_TILE = [{}, {"DSK_GRAPH": "0"}]


@pytest.fixture(autouse=True)
def _release_device_memory():
    """Every test here builds models whose workspaces take up to 9 GiB.  An Engine and its module reference each other,
    so only the cycle collector frees a model and its workspace: run it after each test, and hand the allocator's cached
    blocks back, so that later tests (and the library's own cudaMalloc) get the device memory back."""
    yield
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _env_id(env):
    return "+".join(f"{k}={v}" for k, v in env.items()) or "default"


def _forward(m, x):
    """One forward on a capturable stream (the graph path needs one), synchronised."""
    side, cur = torch.cuda.Stream(), torch.cuda.current_stream()
    side.wait_stream(cur)
    with torch.no_grad(), torch.cuda.stream(side):
        e = m(x).clone()
    cur.wait_stream(side)
    torch.cuda.synchronize()
    return e


def _activations(m, B, T):
    """Per-layer (image (B,C,H,W) on the CPU, pad values) of the handle's last forward."""
    bufs = read_eval_activations(m, B, T, "fp16")
    torch.cuda.synchronize()
    return unpack_eval_activations(m._engine.lib, bufs, B, T)


def _batch_calls(T):
    """(indices into the pool) of each call: a few single utterances, 7, 64, 256, the whole pool, a permuted 256."""
    g = torch.Generator().manual_seed(T)
    perm = torch.randperm(POOL, generator=g)[:256]
    return [torch.tensor([i]) for i in (0, 150, POOL - 1)] + [torch.arange(7), torch.arange(64), torch.arange(256),
                                                               torch.arange(POOL), perm]


def _check_activations(tag, small, large, idx):
    """Each utterance's slice of every activation of the small call equals its slice in the large call."""
    for i, ((a, pa), (b, pb)) in enumerate(zip(small, large)):
        assert float(pa.abs().max()) == 0.0 and float(pb.abs().max()) == 0.0, f"{tag}: a pad of activation {i} is not 0"
        assert torch.equal(a, b[idx]), f"{tag}: activation {i} depends on the batch"


@pytest.mark.parametrize("T", [16, 32, 48, 64, 80, 96, 112, 160, 800])  # T / 16 = 1 ... 7 (odd and even stage-4 heights), 10, 50
@pytest.mark.parametrize("env", WHOLE_TILE, ids=_env_id)
def test_eval_forward_is_batch_invariant(cuda_dev, env, T):
    sd = O.make_state_dict(4, 16)
    pool = O.make_input(POOL, T, 900 + T, 4.0).cuda()
    m = _fresh_model(sd, env)
    big = 64 if T == 800 else POOL                       # the large call whose activations are read back
    ref = _forward(m, pool)
    acts_big = _activations(m, POOL, T) if big == POOL else None
    for idx in _batch_calls(T):
        e = _forward(m, pool[idx.cuda()].contiguous())
        bad = (e != ref[idx.cuda()]).any(dim=1)
        assert not bool(bad.any()), (f"{_env_id(env)} T={T} B={idx.numel()}: {int(bad.sum())} embeddings differ from "
                                     f"the batch of {POOL}, max |diff| {(e - ref[idx.cuda()]).abs().max().item():.3e}")
        if idx.numel() == big and big != POOL and bool((idx == torch.arange(big)).all()):
            acts_big = _activations(m, big, T)
        if idx.numel() == 7:
            acts_small = _activations(m, 7, T)
    _check_activations(f"{_env_id(env)} T={T} 7 vs {big}", acts_small, acts_big, slice(0, 7))
    print(f"{_env_id(env)} T={T}: embeddings and activations bit-identical across batches 1, 7, 64, 256, {POOL}")


@pytest.mark.parametrize("dt,B,T", [("fp16", 256, 160), ("bf16", 256, 160), ("fp16", 257, 160), ("fp16", 2, 4000)])
def test_eval_chain_layer_by_layer_at_serving_shapes(cuda_dev, dt, B, T):
    eval_case(dt, B, T, {})


def _read_conv2(m, B, T):
    """Conv 2's parity-planar output [4][rows][17][64] of the handle's last forward (read_eval_activations for this one
    layer: the long-utterance runs do not have room for a copy of all twelve)."""
    eng = m._engine
    npl = eng.lib.dsk_padded_positions(B, T // 4, 16)
    buf = torch.empty(4, npl // 17, 17, 64, dtype=torch.float16, device="cuda")
    flag = ctypes.c_int32(-1)
    L.check(eng.lib.dsk_debug_read_eval_activation(eng.handle, 2, buf.data_ptr(), buf.numel() * 2, ctypes.byref(flag),
                                                   L.cur_stream()), "dsk_debug_read_eval_activation")
    torch.cuda.synchronize()
    assert flag.value == 1
    return buf


def _planar_slice(buf, n, H, W):
    """Rows of image n in each plane of a parity-planar activation buffer [4][rows][W/2+1][C]."""
    H2 = H // 2
    return buf[:, n * (H2 + 1) + 1:n * (H2 + 1) + 1 + H2]


def _planar_pads(buf, B, H, W):
    """Every element of a parity-planar buffer outside the B images' real pixels."""
    H2 = H // 2
    rows = torch.arange(buf.shape[1], device=buf.device)
    real_row = (rows >= 1) & (rows <= B * (H2 + 1)) & (rows % (H2 + 1) != 0)
    real = real_row.view(-1, 1) & (torch.arange(buf.shape[2], device=buf.device) >= 1).view(1, -1)
    return buf[:, ~real]


@pytest.mark.parametrize("T", [48000, 24000])
def test_long_utterances_past_the_32_bit_reciprocal(cuda_dev, T):
    """B = the smallest batch at which the old reciprocal misplaced a row of conv 2: every embedding equals the
    utterance forwarded alone and in the batch one smaller; conv 2's planar output of the last utterance equals its
    output alone, and every pad is 0."""
    B, (img, h) = first_failing_batch(T)
    assert (B, (img, h)) == OLD_FAILS[T]
    need = eval_workspace(B, T) + 4 * GIB   # the workspace, conv 2 read back, the inputs
    gc.collect()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        print(f"skipped: {free / GIB:.1f} GiB free, the run needs {need / GIB:.1f} GiB")
        pytest.skip(f"{free / GIB:.1f} GiB free < {need / GIB:.1f} GiB")
    sd = O.make_state_dict(4, 16)
    x = O.make_input(B, T, 1100 + B, 4.0).cuda()
    m = _fresh_model(sd, {})
    H, W = T // 2, 32
    e = _forward(m, x)
    act2 = _read_conv2(m, B, T)
    last = _planar_slice(act2, B - 1, H, W).clone()
    pads = _planar_pads(act2, B, H, W)
    nz = int((pads != 0).sum())
    del act2, pads
    e_less = _forward(m, x[:B - 1].contiguous())
    alone = torch.cat([_forward(m, x[i:i + 1].contiguous()) for i in range(B)])
    act2_alone = _read_conv2(m, 1, T)
    diff_alone = (e != alone).any(dim=1).nonzero().flatten().tolist()
    diff_less = (e[:B - 1] != e_less).any(dim=1).nonzero().flatten().tolist()
    print(f"T={T} B={B}: utterances differing from alone {diff_alone}, from the batch of {B - 1} {diff_less}; "
          f"non-zero pads of conv 2 {nz}")
    assert nz == 0, f"{nz} pad elements of conv 2's planar output are not 0"
    assert torch.equal(last, _planar_slice(act2_alone, 0, H, W)), "conv 2 of the last utterance depends on the batch"
    assert not diff_alone and not diff_less


@pytest.mark.parametrize("W", [4, 8])
def test_halo_conv_planar_output_tall(hl, W):  # noqa: F811
    """test_halo_conv_planar_output's case at the tall geometry the old reciprocal got wrong (last row of image 1),
    against the fp64 conv (on the GPU), pads included."""
    lib, h = hl
    N, H = TALL_OP
    C = 64
    g = torch.Generator().manual_seed(W)
    x = torch.randn(N, C, H, W, generator=g) * 2.0
    w = torch.randn(C, C, 3, 3, generator=g) * (2.0 / (9 * C)) ** 0.5
    scale = torch.empty(C).uniform_(0.5, 1.5, generator=g)
    bias = torch.randn(C, generator=g) * 0.1
    res = torch.randn(N, C, H, W, generator=g) * 2.0
    d = lambda t: t.half().double().cuda()
    ref = (F.conv2d(d(x), d(w), None, 1, 1) * scale.double().cuda().view(1, -1, 1, 1)
           + bias.double().cuda().view(1, -1, 1, 1) + d(res)).clamp(0, 20).cpu()
    xp, _ = to_padded(lib, x)
    rp, _ = to_padded(lib, res)
    npl = lib.dsk_padded_positions(N, H // 2, W // 2)
    outp = torch.zeros(4, npl // (W // 2 + 1), W // 2 + 1, C, dtype=torch.float16, device="cuda")
    wd, sc, bi = w.cuda(), scale.cuda(), bias.cuda()
    wp = torch.empty(C * C * 9, dtype=torch.int16, device="cuda")
    s = L.cur_stream()
    L.check(lib.dsk_pack_conv_weight(h, wd.data_ptr(), wp.data_ptr(), C, C, 3, s))
    L.check(lib.dsk_conv3x3_padded(h, xp.data_ptr(), wp.data_ptr(), sc.data_ptr(), bi.data_ptr(), rp.data_ptr(), outp.data_ptr(),
                                   N, H, W, C, 3, 20.0, 1, s), "dsk_conv3x3_padded planar")
    torch.cuda.synchronize()
    got, pads = from_planar(lib, outp, N, C, H, W)
    tol = 2.0 ** -10 * ref.abs().clamp(min=1.0) + 1e-3
    err = (got.double() - ref).abs()
    bad = (err > tol).nonzero()
    assert bad.shape[0] == 0, f"{bad.shape[0]} outputs off, first (n,c,h,w) {tuple(bad[0].tolist())}, max err {float(err.max()):.3g}"
    assert float(pads.abs().max()) == 0.0
