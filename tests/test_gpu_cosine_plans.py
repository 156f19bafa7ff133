"""The tensor-core cosine and Gram ops on fp16 and bf16 engine handles.

A. The all-pairs and batch-hard ops on a bf16 handle (a bf16 Gram, refine bound at u = 1/256) are bit-exact against the
   C oracles and the exact CUDA-core path, also with norms over four decades and gaps on both sides of the bound.
B. AAM-softmax, GE2E, cosine scoring and gallery search run in fp16 whatever the handle's type: a bf16 handle gives the
   fp16 handle's bits.
C. Shapes at the GEMMs' edges (D > 512: a second 512-column launch of the backward products and K = 3D > 1536; C, P and
   N around the 128-row tile and the 512-wide K slices; galleries around the 16384-column search chunk) against fp64.
D. Every plan rebuilt through a script of key changes gives the bits of a freshly created handle, also right after a
   call with NaN inputs under the same key.
E. Rows whose fp16 image overflows (|x| >= 65520) take the exact scan: the tensor-core all-pairs and batch-hard ops
   return the exact path's bits.
"""
import contextlib
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import engine as EN
from oracle import aam_softmax_oracle as A
from oracle import batch_hard_oracle as BH
from oracle import c_oracle as CO
from oracle import ge2e_oracle as G
from oracle import identification_oracle as IO
from oracle import score_norm_oracle as SN
from tests.test_gpu_aam_softmax import _case as _aam_case, _row_rel
from tests.test_gpu_batch_hard import CASES as BH_CASES, _case as _bh_case, _norm10
from tests.test_gpu_ge2e import METHODS, _case as _ge2e_case, _check_backward, _check_cos, _csr, _scalar
from tests.test_gpu_identification import _gallery, _sliced_cosines
from tests.test_gpu_score_norm import COS_GATE, _case as _score_case, _stats_bounds

pytestmark = pytest.mark.gpu

KINDS = {"f16": L.DSK_F16, "bf16": L.DSK_BF16}


def _create(kind):
    h = ctypes.c_void_p()
    L.check(L.load().dsk_create(ctypes.byref(h), 0, KINDS[kind]), "dsk_create")
    return h


def _destroy(h):
    torch.cuda.synchronize()
    L.check(L.load().dsk_destroy(h), "dsk_destroy")


@pytest.fixture(scope="module")
def handles(cuda_dev):
    hs = {kind: _create(kind) for kind in KINDS}
    yield hs
    for h in hs.values():
        _destroy(h)


def _use(mp, h):
    """Route the engine's cosine and Gram wrappers on cuda:0 to the handle h."""
    mp.setitem(EN._AP_HANDLES, 0, h)


@contextlib.contextmanager
def _fresh(mp, kind):
    """A newly created handle of the given type, routed to for the block and destroyed straight after."""
    h = _create(kind)
    old = EN._AP_HANDLES.get(0)
    _use(mp, h)
    try:
        yield
    finally:
        _destroy(h)
        if old is not None:
            _use(mp, old)


def _g(*key):
    return torch.Generator().manual_seed(zlib.crc32("/".join(map(str, key)).encode()))


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _assert_same(got, ref, what=""):
    """Tensors of the same dtype, shape and bits (NaN payloads included)."""
    assert len(got) == len(ref)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert a.dtype == b.dtype and a.shape == b.shape, (what, i)
        assert torch.equal(_bits(a), _bits(b)), (what, i)


def _on_both(handles, mp, fn):
    """fn() on the fp16 handle and on the bf16 handle, which must give the same bits; returns the fp16 handle's."""
    _use(mp, handles["f16"])
    ref = fn()
    _use(mp, handles["bf16"])
    _assert_same(fn(), ref, "bf16 handle vs fp16 handle")
    return ref


# ---- A. bf16 all-pairs and batch-hard, bit-exact ---------------------------------------------------------------------
def _bf16_bound(d2, norm=10.0):
    """The refine kernel's tolerance (allpairs_select_refine_kernel) on a bf16 handle for rows of the given norm when the
    kept candidates reach squared distance d2: 2 dmax r + r^2 plus its small absolute slack."""
    r = (1.0 / 256.0) * 2.0 * norm * 1.01
    dmax = math.sqrt(d2) + r + 1e-3
    return 2.0 * dmax * r + r * r + 1e-5 * 2.0 * norm * norm + 1e-4


def _gap_case(k, factor, D):
    """Row 0: k other-label rows at distance 4 and 20 at distance d2 with d2^2 = 16 + factor * bound(d2^2); all rows of
    norm 10, each neighbour in its own direction, then rotated at random so that the 16-bit images round."""
    d1, d2sq = 4.0, 16.0
    for _ in range(100):
        d2sq = d1 * d1 + factor * _bf16_bound(d2sq)
    rows = [torch.zeros(D, dtype=torch.float64)]
    rows[0][0] = 10.0
    for m, d in enumerate([d1] * k + [math.sqrt(d2sq)] * 20):
        th = 2.0 * math.asin(d / 20.0)
        x = torch.zeros(D, dtype=torch.float64)
        x[0], x[m + 1] = 10.0 * math.cos(th), 10.0 * math.sin(th)
        rows.append(x)
    rows.append(-rows[0])                                     # row 0's positive, at distance 20
    Q, _ = torch.linalg.qr(torch.randn(D, D, generator=_g("rot", k, factor, D), dtype=torch.float64))
    E = (torch.stack(rows) @ Q).float()
    labels = torch.arange(E.shape[0], dtype=torch.int64)
    labels[-1] = 0
    return E, labels


def _a_case(name):
    g = _g("A", name)
    if name in BH_CASES:
        return _bh_case(name)
    if name == "spread_1024x512":                             # norms over four decades
        E = torch.randn(1024, 512, generator=g) * 10.0 ** torch.empty(1024, 1).uniform_(-2.0, 2.0, generator=g)
        return E, (torch.arange(1024) // 16).long()
    if name == "spread_129x64":
        E = torch.randn(129, 64, generator=g) * 10.0 ** torch.empty(129, 1).uniform_(-2.0, 2.0, generator=g)
        return E, (torch.arange(129) % 9).long()
    if name == "1024x64":
        return _norm10(torch.randn(1024, 64, generator=g)), (torch.arange(1024) // 16).long()
    if name == "129x1024":
        return _norm10(torch.randn(129, 1024, generator=g)), (torch.arange(129) % 10).long()
    if name == "1024x1024":
        return _norm10(torch.randn(1024, 1024, generator=g)), (torch.arange(1024) // 16).long()
    if name.startswith("gap"):                                # gap_{above,below}_k{1,4,8}_D{64,128}
        _, side, k, D = name.split("_")
        return _gap_case(int(k[1:]), 1.02 if side == "above" else 0.98, int(D[1:]))
    raise KeyError(name)


A_CASES = BH_CASES + ["spread_1024x512", "spread_129x64", "1024x64", "129x1024", "1024x1024"] + [
    f"gap_{side}_k{k}_D{D}" for side in ("above", "below") for k in (1, 4, 8) for D in (64, 128)]


def _mine(E, labels, exact=False):
    return EN.batch_hard_mine(E, labels, 0.3, exact)[1:]


@pytest.mark.parametrize("name", A_CASES)
def test_allpairs_and_batch_hard_bit_exact_on_both_handles(handles, monkeypatch, name):
    E, labels = _a_case(name)
    Ed, ld = E.cuda(), labels.cuda()
    oloss, opos, oneg, od_ap, od_an, ovalid = BH.batch_hard_triplet(E.numpy(), labels.numpy(), 0.3)
    for k in (1, 4, 8):
        oidx, oval = CO.allpairs_topk(E.numpy(), labels.numpy(), k)
        exact = EN.allpairs_topk(Ed, ld, k, exact_cuda_cores=True)
        assert np.array_equal(exact[0].cpu().numpy(), oidx) and np.array_equal(exact[1].cpu().numpy(), oval)
        for kind in ("bf16", "f16"):
            _use(monkeypatch, handles[kind])
            _assert_same(EN.allpairs_topk(Ed, ld, k), exact, (kind, k))
    exact = _mine(Ed, ld, True)
    loss, pos, neg, d_ap, d_an, valid = (t.cpu().numpy() for t in exact)
    assert np.array_equal(valid, ovalid) and np.array_equal(pos, opos) and np.array_equal(neg, oneg)
    assert np.array_equal(d_ap, od_ap) and np.array_equal(d_an, od_an)
    assert loss[0] == oloss or abs(loss[0] - oloss) <= 1e-6 * abs(oloss)
    for kind in ("bf16", "f16"):
        _use(monkeypatch, handles[kind])
        _assert_same(_mine(Ed, ld), exact, kind)


@pytest.mark.parametrize("kind", ["bf16", "f16"])
def test_batch_hard_select_rows_uneven_ranges(handles, monkeypatch, kind):
    """Anchor ranges of N = 1000 (Npad = 1024), among them (900, 100): its 128-row Gram tile reads E16 rows up to 1028,
    past Npad."""
    g = _g("rows", kind)
    E = _norm10(torch.randn(1000, 512, generator=g)).cuda()
    labels = (torch.arange(1000, device="cuda") // 8).long()
    whole = _mine(E, labels, True)[1:]
    _use(monkeypatch, handles[kind])
    for row0, rows in ((0, 1), (1, 127), (128, 129), (257, 600), (900, 100), (999, 1), (0, 1000)):
        got = EN.batch_hard_select_rows(E, labels, row0, rows)[1:]
        _assert_same(got, [t[row0:row0 + rows] for t in whole], (row0, rows))
        _assert_same(EN.batch_hard_select_rows(E, labels, row0, rows, exact_cuda_cores=True)[1:], got, (row0, rows))


# ---- B. the cosine ops on a bf16 handle: the fp16 handle's bits -------------------------------------------------------
def _aam_run(E, W, y, m=0.2, s=30.0):
    E, W, y = E.cuda(), W.cuda(), y.cuda()
    _, _, _, loss, cos, lse = EN.aam_softmax(E, W, y, m, s)
    gE, gW = EN.aam_softmax_backward(E, W, y, cos, lse, m, s, torch.ones((), device="cuda"))
    return loss, cos, lse, gE, gW


def _ge2e_whole(E, labels, method):
    csr, V = _csr(labels)
    w, b = _scalar(10.0), _scalar(-5.0)
    Ec, loss, cos, rec = EN.ge2e(E.cuda(), csr, V, w, b, method)
    gE, gw, gb = EN.ge2e_backward(Ec, csr, V, w, b, method, cos, rec, torch.ones((), device="cuda"))
    return loss, cos, rec, gE, gw, gb


def _ge2e_ranges(E, labels, method, bounds):
    """The global-batch GE2E ops over the row ranges [bounds[i], bounds[i + 1]): per range cos, rec, row losses, dcos,
    tdc, gw, gb and gE rows, then the mean loss."""
    csr, V = _csr(labels)
    w, b = _scalar(10.0), _scalar(-5.0)
    Ed, gl = E.cuda(), torch.ones((), device="cuda")
    out, dc, td, rl = [], [], [], []
    for row0, row1 in zip(bounds[:-1], bounds[1:]):
        _, cos, rec, row_loss = EN.ge2e_rows(Ed, csr, V, w, b, method, row0, row1 - row0)
        dcos, tdc, gw, gb = EN.ge2e_dcos_rows(cos, rec, csr, V, w, b, method, row0, row1 - row0, gl)
        out += [cos, rec, row_loss, dcos, tdc, gw, gb]
        dc.append(dcos)
        td.append(tdc)
        rl.append(row_loss)
    dcos, tdc = torch.cat(dc), torch.cat(td)
    for row0, row1 in zip(bounds[:-1], bounds[1:]):
        out.append(EN.ge2e_backward_rows(Ed, csr, dcos, tdc, row0, row1 - row0))
    out.append(EN.ge2e_mean(torch.cat(rl), V))
    return out


def _score_run(E, C, k):
    return (EN.cosine_matrix(E, C),) + tuple(EN.cohort_stats(E, C, k))


def test_aam_softmax_bf16_handle_gives_fp16_bits(handles, monkeypatch):
    E, W, y = _aam_case(384, 1211, 512, "arbitrary")
    _on_both(handles, monkeypatch, lambda: _aam_run(E, W, y))


@pytest.mark.parametrize("method", METHODS)
def test_ge2e_bf16_handle_gives_fp16_bits(handles, monkeypatch, method):
    E, labels = _ge2e_case([6] * 64, 512, "arbitrary", 11)
    whole = _on_both(handles, monkeypatch, lambda: _ge2e_whole(E, labels, method))
    parts = _on_both(handles, monkeypatch, lambda: _ge2e_ranges(E, labels, method, [0, 129, 384]))
    # the ranges compose to the whole batch's cosines, gradient and loss
    _assert_same([torch.cat([parts[0], parts[7]]), torch.cat(parts[14:16]), parts[16]],
                 [whole[1], whole[3], whole[0].reshape(1)], "ranges vs whole batch")


def test_scoring_and_search_bf16_handle_give_fp16_bits(handles, monkeypatch):
    E, C = _score_case(700, 5994, 512, "spread")
    _on_both(handles, monkeypatch, lambda: _score_run(E, C, 300))
    Q, Gal = _gallery(130, 20000, 512, 0)
    _on_both(handles, monkeypatch, lambda: EN.cosine_topk(Q, Gal, 10))


# ---- C. shape edges against fp64 (on both handles, which must agree) -------------------------------------------------
def _gate(gate, D):
    """A cosine gate of the tests at D <= 512, at embedding size D.  The gates rest on 22-bit operands plus D/16
    truncating K16 steps of the tensor cores' fp32 accumulation; the second term dominates and grows with D, so above
    512 a gate scales by D / 512 (cosines near 1 at D = 1024 measure up to ~5e-6)."""
    return gate * max(1.0, D / 512)


AAM_EDGES = [(1, 127, 576), (128, 128, 1024), (129, 129, 576), (513, 511, 1024), (128, 512, 576), (129, 513, 1024),
             (513, 513, 576)]


@pytest.mark.parametrize("shape", AAM_EDGES, ids=lambda s: "x".join(map(str, s)))
def test_aam_softmax_edges_vs_fp64(handles, monkeypatch, shape):
    E, W, y = _aam_case(*shape, "norm10")
    loss, cos, lse, gE, gW = _on_both(handles, monkeypatch, lambda: _aam_run(E, W, y))
    oloss, ref_cos, _ = A.forward(E, W, y, 0.2, 30.0)
    dcos = float((cos.double().cpu() - ref_cos).abs().max())
    assert dcos <= _gate(1e-6, shape[2]), dcos
    assert abs(loss.item() - float(oloss)) <= 1e-5 * max(float(oloss), 1.0), (loss.item(), float(oloss))
    rE, rW = A.backward(E, W, y, 0.2, 30.0, cos=cos.cpu())
    eE, eW = _row_rel(gE, rE), _row_rel(gW, rW)
    assert eE <= 1e-5 and eW <= 1e-5, (eE, eW)


def _counts(N, P):
    return [N // P + (p < N % P) for p in range(P)]


GE2E_EDGES = [(129, 128, 1024), (513, 127, 576), (513, 128, 1024), (513, 129, 576), (1026, 511, 1024),
              (1026, 512, 576), (1026, 513, 1024)]   # (N, P, D)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("shape", GE2E_EDGES, ids=lambda s: "x".join(map(str, s)))
def test_ge2e_edges_vs_fp64(handles, monkeypatch, shape, method):
    N, P, D = shape
    E, labels = _ge2e_case(_counts(N, P), D, "norm10", zlib.crc32(f"edge{shape}".encode()))

    def run():
        _, _, _, loss, cos, rec, gE, gw, gb = _check_backward(E, labels, 10.0, -5.0, method, report=False)
        return loss.reshape(1), cos, rec, gE, gw, gb

    loss, cos, rec, *_ = _on_both(handles, monkeypatch, run)
    oloss, ref_cos, _ = G.forward(E, labels, 10.0, -5.0, method)
    # the cosines come from the scoring GEMM; a singleton's cosine to its own centroid is ~1, where the truncation
    # term is largest, so the non-target cosines are held to the scoring ops' gate
    _check_cos(cos, ref_cos, labels, tol=_gate(COS_GATE, D))
    assert abs(loss.item() - float(oloss)) <= 1e-5 * max(float(oloss), 1.0), (loss.item(), float(oloss))


@pytest.mark.parametrize("M,Nc,D,kind", [(1, 128, 576, "norm10"), (128, 129, 1024, "clustered"),
                                         (129, 128, 1024, "spread"), (513, 129, 576, "norm10")])
def test_scoring_edges_vs_fp64(handles, monkeypatch, M, Nc, D, kind):
    E, C = _score_case(M, Nc, D, kind)
    cos, mean, std = _on_both(handles, monkeypatch, lambda: _score_run(E, C, 50))
    err = float((cos.double() - SN.cosine_matrix(E, C)).abs().max())
    assert err <= _gate(COS_GATE, D), err
    _use(monkeypatch, handles["bf16"])
    for k in (2, 50, Nc):
        eps, *_, dm, ds, tol_m, tol_s = _stats_bounds(E, C, k)
        assert eps <= _gate(COS_GATE, D) and (dm <= tol_m).all() and (ds <= tol_s).all(), k


@pytest.mark.parametrize("Ng", [16383, 16384, 16385])
def test_search_edges_vs_fp64(handles, monkeypatch, Ng):
    Q, Gal = _gallery(129, Ng, 1024, 3)
    for k in (1, 10):
        idx, val = _on_both(handles, monkeypatch, lambda: EN.cosine_topk(Q, Gal, k))
        ri, rv = IO.topk_keys(_sliced_cosines(Q, Gal), k)
        assert torch.equal(idx, ri) and torch.equal(_bits(val), _bits(rv)), k
        Qn, Gn = (X.double() / X.double().norm(dim=1, keepdim=True).clamp_min(1e-300) for X in (Q, Gal))
        err = float((val.double() - torch.gather(Qn @ Gn.T, 1, idx)).abs().max())
        assert err <= _gate(COS_GATE, 1024), (k, err)
    if Ng > 16384:   # a copy of column 16383 sits at 16384, in the next chunk: the tie goes to the lower column
        assert EN.cosine_topk(Q[:1], Gal, 2)[0][0].tolist() == [16383, 16384]


# ---- D. plan lifecycle ----------------------------------------------------------------------------------------------
def _op_allpairs(N, D, row0, rows):
    E = _norm10(torch.randn(N, D, generator=_g("ap", N, D))).cuda()
    lab = (torch.arange(N, device="cuda") // 4).long()
    if (row0, rows) == (0, N):
        return EN.allpairs_topk(E, lab, 8) + _mine(E, lab)
    return EN.batch_hard_select_rows(E, lab, row0, rows)[1:]


def _op_aam(N, C, D, poison=False):
    E, W, y = _aam_case(N, C, D, "norm10")
    if poison:
        E[N // 2] = float("nan")
    return _aam_run(E, W, y)


def _op_ge2e(N, P, D, row0, rows):
    E, labels = _ge2e_case(_counts(N, P), D, "norm10", zlib.crc32(f"life{N}/{P}/{D}".encode()))
    if (row0, rows) == (0, N):
        return _ge2e_whole(E, labels, "softmax")
    csr, V = _csr(labels)
    return EN.ge2e_rows(E.cuda(), csr, V, _scalar(10.0), _scalar(-5.0), "contrast", row0, rows)[1:]


def _op_score(Nc, D, M, poison=False):
    g = _g("score", Nc, D, M)
    E, C = torch.randn(M, D, generator=g).cuda(), torch.randn(Nc, D, generator=g).cuda()
    if poison:
        E[M // 2] = float("nan")
        return (EN.cosine_matrix(E, C),)
    return _score_run(E, C, 20)


def _op_search(Ng, D, M):
    Q, Gal = _gallery(M, Ng, D, 7)
    return EN.cosine_topk(Q, Gal, 10)


OPS = {"allpairs": _op_allpairs, "aam": _op_aam, "ge2e": _op_ge2e, "score": _op_score, "search": _op_search}

# Consecutive steps of one plan change one component of its key, or return to an earlier key.  Plan keys: all-pairs
# (N, D, row0, rows); AAM (N, C, D); GE2E (N, P, D, row0, rows); scoring and search (Nc, D, chunk), the chunk set by M
# (128-row multiples) and the search's Nc by Ng (min(Ng, 16384)).
SCRIPT = [
    ("allpairs", (384, 192, 0, 384)), ("aam", (200, 300, 128)), ("ge2e", (300, 100, 128, 0, 300)),
    ("score", (300, 128, 100)), ("search", (1000, 128, 50)),
    ("allpairs", (384, 192, 0, 128)),                       # rows
    ("aam", (200, 513, 128)),                               # C: a second 512-wide K slice of gE^
    ("ge2e", (300, 100, 128, 0, 150)),                      # rows
    ("score", (300, 128, 200)),                             # M: chunk 128 -> 256
    ("search", (16385, 128, 50)),                           # Ng: Nc 1000 -> 16384, two gallery chunks
    ("allpairs", (384, 192, 64, 128)),                      # row0
    ("aam", (200, 513, 576)),                               # D: two 512-column launches of the backward GEMMs
    ("ge2e", (300, 100, 128, 100, 150)),                    # row0
    ("score", (129, 128, 200)),                             # Nc
    ("search", (16385, 128, 300)),                          # M: chunk 128 -> 384
    ("allpairs", (384, 128, 64, 128)),                      # D
    ("aam", (129, 513, 576)),                               # N
    ("ge2e", (300, 120, 128, 100, 150)),                    # P
    ("score", (129, 192, 200)),                             # D
    ("search", (16384, 128, 300)),                          # Ng: one chunk, same key
    ("allpairs", (256, 128, 64, 128)),                      # N
    ("aam", (200, 300, 128)),                               # back to the first key
    ("ge2e", (300, 120, 192, 100, 150)),                    # D
    ("score", (300, 128, 100)),                             # back to the first key
    ("search", (16384, 192, 300)),                          # D
    ("allpairs", (256, 128, 64, 192)),                      # rows: row0 + rows_pad = 320 > Npad = 256
    ("ge2e", (330, 120, 192, 100, 150)),                    # N
    ("search", (1000, 128, 50)),                            # back to the first key
    ("allpairs", (384, 192, 0, 384)),                       # back to the first key
    ("ge2e", (300, 100, 128, 0, 300)),                      # back to the first key
]


@pytest.mark.parametrize("kind", ["f16", "bf16"])
def test_plan_lifecycle_matches_fresh_handles(handles, monkeypatch, kind):
    shared = handles[kind]
    for op, key in SCRIPT:
        _use(monkeypatch, shared)
        got = OPS[op](*key)
        with _fresh(monkeypatch, kind):
            ref = OPS[op](*key)
        _assert_same(got, ref, (kind, op, key))
    # a call with a NaN row leaves nothing in the cached buffers of its key: the next clean call is the fresh result
    for op, key in (("score", (300, 128, 100)), ("aam", (200, 300, 128))):
        with _fresh(monkeypatch, kind):
            ref = OPS[op](*key)
        _use(monkeypatch, shared)
        poisoned = OPS[op](*key, poison=True)
        assert bool(torch.isnan(poisoned[0]).any()), op
        _assert_same(OPS[op](*key), ref, (kind, op, "after NaN"))


# ---- E. fp16 overflow of the Gram's operands ------------------------------------------------------------------------
def _overflow_case(N, D):
    """N - 10 rows of label 0 and 10 rows of labels 1..10, so a label-0 anchor has 10 valid columns (8 <= 10 < 16).  Three
    of those have one entry of 7e4 and one has norm 1e6 (in fp16: inf); so do two label-0 anchors."""
    E = _norm10(torch.randn(N, D, generator=_g("overflow", N, D)))
    labels = torch.cat([torch.zeros(N - 10), torch.arange(1, 11)]).long()
    E[N - 3:, 5] = 7e4
    E[N - 10] *= 1e5
    E[0, 3] = 7e4
    E[1] *= 1e5
    return E, labels


@pytest.mark.parametrize("N,D", [(40, 64), (40, 1024), (1100, 64)])
def test_overflowing_rows_take_the_exact_scan(handles, monkeypatch, N, D):
    E, labels = _overflow_case(N, D)
    Ed, ld = E.cuda(), labels.cuda()
    _use(monkeypatch, handles["f16"])
    for k in (1, 4, 8):
        exact = EN.allpairs_topk(Ed, ld, k, exact_cuda_cores=True)
        got = EN.allpairs_topk(Ed, ld, k)
        bad = (got[0] != exact[0]).any(dim=1) | (_bits(got[1]) != _bits(exact[1])).any(dim=1)
        assert not bool(bad.any()), (k, bad.nonzero().flatten().tolist()[:8], got[0][bad][:2].tolist())
    exact = _mine(Ed, ld, True)
    got = _mine(Ed, ld)
    _assert_same(got[1:], exact[1:], "selection")       # before any index reaches the backward
    _assert_same(got[:1], exact[:1], "loss")
    _, pos, neg, d_ap, d_an, valid = exact
    assert bool((neg[valid] >= 0).all()) and bool((pos[valid] >= 0).all())
    gl = torch.ones((), device="cuda")
    _assert_same([EN.batch_hard_backward(Ed, *got[1:], 0.3, gl)], [EN.batch_hard_backward(Ed, *exact[1:], 0.3, gl)])
