"""Host-side engine: owns the libdsk handle of one DeepSpeakerModel, keeps the repacked weights in sync
with the nn.Parameters, and wraps the C-ABI calls in torch.autograd.Functions.

PyTorch is plumbing here (device memory, streams, autograd graph); all arithmetic is in libdsk.so.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from . import _lib as L

_CONV_ORDER = None


def conv_bn_modules(model):
    """The 12 (conv, bn) pairs in C-ABI order: i = 3*stage + {0: convK/bnK, 1: layerK.0.conv1/bn1, 2: conv2/bn2}."""
    m = model.model
    out = []
    for s in range(1, 5):
        blk = getattr(m, f"layer{s}")[0]
        out += [(getattr(m, f"conv{s}"), getattr(m, f"bn{s}")), (blk.conv1, blk.bn1), (blk.conv2, blk.bn2)]
    return out


def _f32c(t):
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise RuntimeError("libdsk needs contiguous float32 CUDA tensors")
    return t


class Engine:
    def __init__(self, module, device, operand_dtype, share_from=None):
        """``share_from``: another Engine of the same module whose packed weights this one borrows (inference lanes of
        ``EmbeddingPipeline``: one weight image in L2 for all forwards in flight)."""
        if device.type != "cuda":
            raise RuntimeError("the H100 engine runs on CUDA devices only")
        self.lib = L.load()
        self.device = device
        self.index = device.index if device.index is not None else torch.cuda.current_device()
        self.module_ref = module  # plain reference; Engine lifetime == module lifetime
        self.handle = ctypes.c_void_p()
        L.check(self.lib.dsk_create(ctypes.byref(self.handle), self.index,
                                    L.DSK_BF16 if operand_dtype == "bf16" else L.DSK_F16), "dsk_create")
        self._versions = None
        self._wstruct = None
        self.train_calls = 0  # train-mode forwards update BN running stats through raw pointers
        self.side_streams = []  # forward_train_many: one stream per forward in flight
        self._gscratch, self._gslot = [], 0
        self.bucket_accumulations = 0  # backwards that added their gradients straight into an optimizer bucket
        self.share_from = share_from
        if share_from is not None:
            L.check(self.lib.dsk_share_weights(self.handle, share_from.handle), "dsk_share_weights")

    def set_loss_scale(self, scale: float):
        """fp16 gradient scale used inside the backward (0 = automatic, see include/dsk.h)."""
        L.check(self.lib.dsk_set_loss_scale(self.handle, float(scale)), "dsk_set_loss_scale")

    def __del__(self):
        try:
            if getattr(self, "handle", None) and self.handle.value:
                self.lib.dsk_destroy(self.handle)
                self.handle = ctypes.c_void_p()
        except Exception:
            pass

    # -- parameters ---------------------------------------------------------------------------------
    def _param_versions(self, eval_mode):
        m = self.module_ref
        vs = []
        for conv, bn in conv_bn_modules(m):
            vs += [conv.weight._version, conv.weight.data_ptr(), bn.weight._version, bn.bias._version]
            if eval_mode:
                vs += [bn.running_mean._version, bn.running_var._version]
        fc = m.model.fc
        vs += [fc.weight._version, fc.bias._version, fc.weight.data_ptr(), int(eval_mode),
               self.train_calls if eval_mode else 0]
        return tuple(vs)

    def invalidate(self):
        """Force a repack / BN re-fold at the next forward.  Change detection relies on ``tensor._version`` (bumped by
        every in-place op on the parameter itself, which is what optimizers and ``load_state_dict`` do) and on
        ``data_ptr``; writes through ``param.data`` / ``buffer.data`` (``p.data.fill_()``, ``p.data.copy_()``, the
        reference's init idiom, model.py:114-120) do NOT bump the version: call this (or
        ``DeepSpeakerModel.refresh_weights()``) after such a write."""
        self._versions = None

    def sync_weights(self, eval_mode=True):
        """Repack/fold when any parameter (or, in eval, BN buffer) changed since the last call (see ``invalidate``)."""
        if self.share_from is not None:
            if not eval_mode:
                raise RuntimeError("an engine that borrows its weights is inference-only")
            self.share_from.sync_weights(True)
            return
        vs = self._param_versions(eval_mode)
        if vs == self._versions:
            return
        m = self.module_ref
        w = L.DskWeights()
        for i, (conv, bn) in enumerate(conv_bn_modules(m)):
            for t in (conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var):
                if not t.is_cuda or t.device != self.device:
                    raise RuntimeError("model parameters must live on the engine's CUDA device (call model.cuda())")
            w.conv_w[i] = _f32c(conv.weight.data).data_ptr()
            w.bn_gamma[i] = _f32c(bn.weight.data).data_ptr()
            w.bn_beta[i] = _f32c(bn.bias.data).data_ptr()
            w.bn_running_mean[i] = _f32c(bn.running_mean).data_ptr()
            w.bn_running_var[i] = _f32c(bn.running_var).data_ptr()
        w.fc_w = _f32c(m.model.fc.weight.data).data_ptr()
        w.fc_b = _f32c(m.model.fc.bias.data).data_ptr()
        w.embedding_size = m.embedding_size
        self._wstruct = w
        if eval_mode:
            L.check(self.lib.dsk_load_weights(self.handle, ctypes.byref(w), L.cur_stream()), "dsk_load_weights")
        else:   # once per training step: only the operand images the training path reads, in one launch
            L.check(self.lib.dsk_load_weights_train(self.handle, ctypes.byref(w), L.cur_stream()), "dsk_load_weights_train")
        self._versions = vs

    def grad_scratch(self, params, slots: int = 6, with_flat: bool = False):
        """Per-parameter gradient tensors for one backward, as views of a flat scratch buffer that is allocated once and
        rotated over ``slots`` buffers (a backward allocated 38 tensors per call: ~0.2 ms of host time per context, and
        the training step is host-sensitive - ~450 kernel launches per 7 ms of GPU work).  Safe to recycle: a slot is
        reused ``slots`` backwards later, and autograd has consumed a backward's gradients (added them into ``p.grad`` on
        the stream the next step is ordered after) long before that."""
        key = tuple((p.data_ptr(), p.numel()) for p in params)
        if not self._gscratch or self._gscratch[0][0] != key:
            total = sum((p.numel() + 3) // 4 * 4 for p in params)
            self._gscratch = []
            for _ in range(slots):
                flat = torch.empty(total, device=self.device, dtype=torch.float32)
                views, off = [], 0
                for p in params:
                    views.append(flat[off:off + p.numel()].view_as(p))
                    off += (p.numel() + 3) // 4 * 4
                self._gscratch.append((key, flat, views))
            self._gslot = 0
        _, flat, views = self._gscratch[self._gslot]
        self._gslot = (self._gslot + 1) % len(self._gscratch)
        return (flat, views) if with_flat else views

    # -- forward ------------------------------------------------------------------------------------
    def forward(self, x, training):
        x = x.contiguous()
        if x.dtype != torch.float32:
            x = x.float()
        B, _, T, _ = x.shape
        with torch.cuda.device(self.device):
            if training:
                from . import train as _train  # batch-statistics BN + autograd path

                return _train.forward_train(self, x)
            self.sync_weights(eval_mode=True)
            emb = torch.empty(B, self.module_ref.embedding_size, device=x.device, dtype=torch.float32)
            L.check(self.lib.dsk_rescnn_forward(self.handle, x.data_ptr(), B, T, emb.data_ptr(), L.DSK_EVAL,
                                                L.cur_stream()), "dsk_rescnn_forward")
        return emb


# ---------------------------------------------------------------------------------------------------
# distances / loss / selection
# ---------------------------------------------------------------------------------------------------
def _check2d(*ts):
    for t in ts:
        if not t.is_cuda:
            raise RuntimeError("libdsk distance/loss ops need CUDA tensors; there is no CPU fallback")
        if t.dim() != 2:
            raise RuntimeError("expected (B, D) tensors")


class PairwiseDistanceFn(torch.autograd.Function):
    """PairwiseDistance(2).forward — reference model.py:13-18."""

    @staticmethod
    def forward(ctx, x1, x2):
        _check2d(x1, x2)
        x1c, x2c = x1.detach().float().contiguous(), x2.detach().float().contiguous()
        B, D = x1c.shape
        out = torch.empty(B, device=x1.device, dtype=torch.float32)
        with torch.cuda.device(x1.device):
            L.check(L.load().dsk_pairwise_distance(x1c.data_ptr(), x2c.data_ptr(), B, D, out.data_ptr(), L.cur_stream()),
                    "dsk_pairwise_distance")
        ctx.save_for_backward(x1c, x2c, out)
        return out

    @staticmethod
    def backward(ctx, go):
        x1, x2, dist = ctx.saved_tensors
        B, D = x1.shape
        go = go.float().contiguous()
        g1 = torch.empty_like(x1) if ctx.needs_input_grad[0] else None
        g2 = torch.empty_like(x2) if ctx.needs_input_grad[1] else None
        with torch.cuda.device(x1.device):
            L.check(L.load().dsk_pairwise_distance_bwd(x1.data_ptr(), x2.data_ptr(), dist.data_ptr(), go.data_ptr(), B, D,
                                                       L.ptr(g1), L.ptr(g2), L.cur_stream()), "dsk_pairwise_distance_bwd")
        return g1, g2


class TripletLossFn(torch.autograd.Function):
    """TripletMarginLoss(margin).forward — reference model.py:27-33 (loss is a device scalar)."""

    @staticmethod
    def forward(ctx, a, p, n, margin):
        _check2d(a, p, n)
        ac, pc, nc = (t.detach().float().contiguous() for t in (a, p, n))
        B, D = ac.shape
        loss = torch.empty(1, device=a.device, dtype=torch.float32)
        d_p = torch.empty(B, device=a.device, dtype=torch.float32)
        d_n = torch.empty(B, device=a.device, dtype=torch.float32)
        with torch.cuda.device(a.device):
            L.check(L.load().dsk_triplet_loss(ac.data_ptr(), pc.data_ptr(), nc.data_ptr(), B, D, margin, loss.data_ptr(),
                                              d_p.data_ptr(), d_n.data_ptr(), L.cur_stream()), "dsk_triplet_loss")
        ctx.save_for_backward(ac, pc, nc, d_p, d_n)
        ctx.margin = margin
        return loss.reshape(())

    @staticmethod
    def backward(ctx, gl):
        a, p, n, d_p, d_n = ctx.saved_tensors
        B, D = a.shape
        gl = gl.float().reshape(1).contiguous()
        ga, gp, gn = torch.empty_like(a), torch.empty_like(p), torch.empty_like(n)
        with torch.cuda.device(a.device):
            L.check(L.load().dsk_triplet_loss_bwd(a.data_ptr(), p.data_ptr(), n.data_ptr(), d_p.data_ptr(), d_n.data_ptr(),
                                                  gl.data_ptr(), B, D, ctx.margin, ga.data_ptr(), gp.data_ptr(),
                                                  gn.data_ptr(), L.cur_stream()), "dsk_triplet_loss_bwd")
        return ga, gp, gn, None


def margin_select(d_p, d_n, margin):
    _ = [t for t in (d_p, d_n) if not t.is_cuda and (_ for _ in ()).throw(RuntimeError("CUDA tensors required"))]
    d_p, d_n = d_p.detach().float().contiguous(), d_n.detach().float().contiguous()
    B = d_p.numel()
    idx = torch.empty(B, device=d_p.device, dtype=torch.int64)
    count = torch.empty(1, device=d_p.device, dtype=torch.int32)
    with torch.cuda.device(d_p.device):
        L.check(L.load().dsk_margin_select(d_p.data_ptr(), d_n.data_ptr(), B, float(margin), idx.data_ptr(),
                                           count.data_ptr(), L.cur_stream()), "dsk_margin_select")
    return idx, count


def gather_rows(src, idx, count):
    """out[j] = src[idx[j]] for j < count (train_triplet.py:265-274), rows beyond count are left untouched."""
    src = src.detach().float().contiguous()
    rows = src.shape[0]
    row_elems = src[0].numel()
    out = torch.zeros_like(src)
    with torch.cuda.device(src.device):
        L.check(L.load().dsk_gather_rows(src.data_ptr(), idx.data_ptr(), count.data_ptr(), rows, row_elems,
                                         out.data_ptr(), L.cur_stream()), "dsk_gather_rows")
    return out


_AP_HANDLES = {}


def _allpairs_handle(device):
    """Module-level fp16 engine handle for the tensor-core all-pairs, AAM-softmax and cosine-scoring ops (one per
    device)."""
    key = device.index if device.index is not None else torch.cuda.current_device()
    if key not in _AP_HANDLES:
        h = ctypes.c_void_p()
        L.check(L.load().dsk_create(ctypes.byref(h), key, L.DSK_F16), "dsk_create")
        _AP_HANDLES[key] = h
    return _AP_HANDLES[key]


def allpairs_topk(E, labels, k, exact_cuda_cores: bool = False):
    """exact_cuda_cores=True forces the all-fp32 CUDA-core path; the default tensor-core path returns the same bits."""
    if not E.is_cuda:
        raise RuntimeError("CUDA tensors required")
    E = E.detach().float().contiguous()
    labels = labels.to(device=E.device, dtype=torch.int64).contiguous()
    N, D = E.shape
    idx = torch.empty(N, k, device=E.device, dtype=torch.int64)
    val = torch.empty(N, k, device=E.device, dtype=torch.float32)
    with torch.cuda.device(E.device):
        if exact_cuda_cores:
            L.check(L.load().dsk_allpairs_topk(E.data_ptr(), labels.data_ptr(), N, D, k, idx.data_ptr(), val.data_ptr(),
                                               L.cur_stream()), "dsk_allpairs_topk")
        else:
            L.check(L.load().dsk_allpairs_topk_tc(_allpairs_handle(E.device), E.data_ptr(), labels.data_ptr(), N, D, k,
                                                  idx.data_ptr(), val.data_ptr(), L.cur_stream()), "dsk_allpairs_topk_tc")
    return idx, val


def batch_hard_mine(E, labels, margin, exact_cuda_cores: bool = False):
    """dsk_batch_hard_triplet: (loss (1,), pos_idx, neg_idx, d_ap, d_an, valid (bool)) on E's device.  The default
    tensor-core Gram path and ``exact_cuda_cores=True`` return the same bits."""
    _check2d(E)
    E = E.detach().float().contiguous()
    labels = labels.to(device=E.device, dtype=torch.int64).contiguous()
    N, D = E.shape
    if labels.shape != (N,):
        raise RuntimeError(f"expected labels of shape ({N},), got {tuple(labels.shape)}")
    dev = E.device
    loss = torch.empty(1, device=dev, dtype=torch.float32)
    pos, neg = (torch.empty(N, device=dev, dtype=torch.int64) for _ in range(2))
    d_ap, d_an = (torch.empty(N, device=dev, dtype=torch.float32) for _ in range(2))
    valid = torch.empty(N, device=dev, dtype=torch.bool)
    with torch.cuda.device(dev):
        h = None if exact_cuda_cores else _allpairs_handle(dev)
        L.check(L.load().dsk_batch_hard_triplet(h, E.data_ptr(), labels.data_ptr(), N, D, float(margin), loss.data_ptr(),
                                                pos.data_ptr(), neg.data_ptr(), d_ap.data_ptr(), d_an.data_ptr(),
                                                valid.data_ptr(), L.cur_stream()), "dsk_batch_hard_triplet")
    return E, loss, pos, neg, d_ap, d_an, valid


def batch_hard_backward(E, pos, neg, d_ap, d_an, valid, margin, grad_loss):
    """dsk_batch_hard_triplet_bwd: d loss / d E scaled by the device scalar ``grad_loss``."""
    N, D = E.shape
    gl = grad_loss.float().reshape(1).contiguous()
    gE = torch.empty_like(E)
    with torch.cuda.device(E.device):
        L.check(L.load().dsk_batch_hard_triplet_bwd(E.data_ptr(), pos.data_ptr(), neg.data_ptr(), d_ap.data_ptr(),
                                                    d_an.data_ptr(), N, D, float(margin), gl.data_ptr(), valid.data_ptr(),
                                                    gE.data_ptr(), L.cur_stream()), "dsk_batch_hard_triplet_bwd")
    return gE


def batch_hard_select_rows(E, labels, row0, rows, exact_cuda_cores: bool = False):
    """dsk_batch_hard_select_rows: the selection of the anchors [row0, row0 + rows) of the batch E (N, D) ->
    (E fp32 contiguous, pos_idx, neg_idx, d_ap, d_an, valid (bool)), each (rows,) on E's device, bit-identical to those
    rows of ``batch_hard_mine``.  Indices are global.  The tensor-core Gram plan is cached per (N, D, row0, rows)."""
    _check2d(E)
    E = E.detach().float().contiguous()
    labels = labels.to(device=E.device, dtype=torch.int64).contiguous()
    N, D = E.shape
    if labels.shape != (N,):
        raise RuntimeError(f"expected labels of shape ({N},), got {tuple(labels.shape)}")
    dev, n = E.device, max(int(rows), 0)
    pos, neg = (torch.empty(n, device=dev, dtype=torch.int64) for _ in range(2))
    d_ap, d_an = (torch.empty(n, device=dev, dtype=torch.float32) for _ in range(2))
    valid = torch.empty(n, device=dev, dtype=torch.bool)
    with torch.cuda.device(dev):
        h = None if exact_cuda_cores else _allpairs_handle(dev)
        L.check(L.load().dsk_batch_hard_select_rows(h, E.data_ptr(), labels.data_ptr(), N, D, int(row0), int(rows),
                                                    pos.data_ptr(), neg.data_ptr(), d_ap.data_ptr(), d_an.data_ptr(),
                                                    valid.data_ptr(), L.cur_stream()), "dsk_batch_hard_select_rows")
    return E, pos, neg, d_ap, d_an, valid


def batch_hard_mean(d_ap, d_an, valid, margin):
    """dsk_batch_hard_mean: loss (1,) from the selection of all N anchors, the bits of ``batch_hard_mine``'s loss."""
    N = d_ap.shape[0]
    loss = torch.empty(1, device=d_ap.device, dtype=torch.float32)
    with torch.cuda.device(d_ap.device):
        L.check(L.load().dsk_batch_hard_mean(d_ap.data_ptr(), d_an.data_ptr(), valid.data_ptr(), N, float(margin),
                                             loss.data_ptr(), L.cur_stream()), "dsk_batch_hard_mean")
    return loss


def batch_hard_backward_rows(E, pos, neg, d_ap, d_an, valid, row0, rows, margin, grad_loss):
    """dsk_batch_hard_triplet_bwd_rows: rows [row0, row0 + rows) of ``batch_hard_backward`` -> (rows, D), the same
    bits.  The selection tensors cover all N anchors of E."""
    N, D = E.shape
    gl = grad_loss.float().reshape(1).contiguous()
    gE = torch.empty(max(int(rows), 0), D, device=E.device, dtype=torch.float32)
    with torch.cuda.device(E.device):
        L.check(L.load().dsk_batch_hard_triplet_bwd_rows(E.data_ptr(), pos.data_ptr(), neg.data_ptr(), d_ap.data_ptr(),
                                                         d_an.data_ptr(), valid.data_ptr(), N, D, int(row0), int(rows),
                                                         float(margin), gl.data_ptr(), gE.data_ptr(), L.cur_stream()),
                "dsk_batch_hard_triplet_bwd_rows")
    return gE


class BatchHardTripletFn(torch.autograd.Function):
    """Batch-hard triplet loss (in-batch hardest positive and negative per anchor, mean hinge over valid anchors);
    the loss is a device scalar."""

    @staticmethod
    def forward(ctx, E, labels, margin, exact_cuda_cores):
        Ec, loss, pos, neg, d_ap, d_an, valid = batch_hard_mine(E, labels, margin, exact_cuda_cores)
        ctx.save_for_backward(Ec, pos, neg, d_ap, d_an, valid)
        ctx.margin = margin
        return loss.reshape(())

    @staticmethod
    def backward(ctx, gl):
        E, pos, neg, d_ap, d_an, valid = ctx.saved_tensors
        return batch_hard_backward(E, pos, neg, d_ap, d_an, valid, ctx.margin, gl), None, None, None


# ---------------------------------------------------------------------------------------------------
# additive angular margin softmax
# ---------------------------------------------------------------------------------------------------
def _aam_inputs(E, W, labels):
    for t in (E, W):
        if not t.is_cuda:
            raise RuntimeError("the AAM-softmax loss needs CUDA tensors; there is no CPU fallback")
    if E.dim() != 2 or W.dim() != 2 or E.shape[1] != W.shape[1]:
        raise RuntimeError(f"expected embeddings (N, D) and weight (C, D), got {tuple(E.shape)} and {tuple(W.shape)}")
    if W.device != E.device:
        raise RuntimeError("embeddings and weight must be on one device")
    E = E.detach().float().contiguous()
    W = W.detach().float().contiguous()
    labels = torch.as_tensor(labels).to(device=E.device, dtype=torch.int64).contiguous()
    if labels.shape != (E.shape[0],):
        raise RuntimeError(f"expected labels of shape ({E.shape[0]},), got {tuple(labels.shape)}")
    return E, W, labels


def aam_subcentre_args(rows, subcentres, topk, topk_margin):
    """Checks the sub-centre arguments for a (C K, D) weight of ``rows`` rows and returns C: ValueError unless
    1 <= K <= 16, K divides the rows, 0 <= topk <= min(C - 1, 64) and m' is finite and >= 0.  C >= 2 and
    C K <= 65536 are the op's own checks."""
    K = subcentres
    if isinstance(K, bool) or not isinstance(K, int) or not 1 <= K <= L.DSK_AAM_MAX_SUBCENTRES:
        raise ValueError(f"subcentres must be an int in [1, {L.DSK_AAM_MAX_SUBCENTRES}], got {K!r}")
    if rows % K:
        raise ValueError(f"the weight must have C * subcentres rows; {rows} rows are not a multiple of {K}")
    C = rows // K
    if isinstance(topk, bool) or not isinstance(topk, int) or topk < 0 or \
            (topk > 0 and topk > min(C - 1, L.DSK_AAM_MAX_TOPK)):
        raise ValueError(f"topk must be an int in [0, min(C - 1, {L.DSK_AAM_MAX_TOPK})] with C = {C}, got {topk!r}")
    if not math.isfinite(float(topk_margin)) or float(topk_margin) < 0.0:
        raise ValueError(f"topk_margin must be finite and >= 0, got {topk_margin!r}")
    return C


def aam_softmax_sc(E, W, labels, margin, scale, subcentres=1, topk=0, topk_margin=0.0):
    """dsk_aam_softmax_sc: (E, W, labels as the op read them, loss (1,), cos (N, C), lse (N,), sub (N, C) uint8 or
    None when subcentres = 1, top (N, topk) int32 or None when topk = 0) on E's device.  W is (C * subcentres, D)."""
    E, W, labels = _aam_inputs(E, W, labels)
    C = aam_subcentre_args(W.shape[0], subcentres, topk, topk_margin)
    N, D = E.shape
    dev = E.device
    loss = torch.empty(1, device=dev, dtype=torch.float32)
    cos = torch.empty(N, C, device=dev, dtype=torch.float32)
    lse = torch.empty(N, device=dev, dtype=torch.float32)
    sub = torch.empty(N, C, device=dev, dtype=torch.uint8) if subcentres > 1 else None
    top = torch.empty(N, topk, device=dev, dtype=torch.int32) if topk > 0 else None
    with torch.cuda.device(dev):
        L.check(L.load().dsk_aam_softmax_sc(_allpairs_handle(dev), E.data_ptr(), W.data_ptr(), labels.data_ptr(), N, C,
                                            subcentres, D, float(margin), float(scale), topk, float(topk_margin),
                                            loss.data_ptr(), cos.data_ptr(), lse.data_ptr(), L.ptr(sub), L.ptr(top),
                                            L.cur_stream()), "dsk_aam_softmax_sc")
    return E, W, labels, loss, cos, lse, sub, top


def aam_softmax_sc_backward(E, W, labels, cos, lse, sub, top, margin, scale, subcentres, topk, topk_margin, grad_loss):
    """dsk_aam_softmax_sc_bwd: (gE (N, D), gW (C * subcentres, D)) = d loss / d (E, W) scaled by the device scalar
    ``grad_loss``, from the forward's cos, lse, sub and top."""
    N, D = E.shape
    C = aam_subcentre_args(W.shape[0], subcentres, topk, topk_margin)
    gl = grad_loss.float().reshape(1).contiguous()
    gE, gW = torch.empty_like(E), torch.empty_like(W)
    with torch.cuda.device(E.device):
        L.check(L.load().dsk_aam_softmax_sc_bwd(_allpairs_handle(E.device), E.data_ptr(), W.data_ptr(),
                                                labels.data_ptr(), cos.data_ptr(), lse.data_ptr(), L.ptr(sub),
                                                L.ptr(top), N, C, subcentres, D, float(margin), float(scale), topk,
                                                float(topk_margin), gl.data_ptr(), gE.data_ptr(), gW.data_ptr(),
                                                L.cur_stream()), "dsk_aam_softmax_sc_bwd")
    return gE, gW


def aam_softmax(E, W, labels, margin, scale):
    """dsk_aam_softmax: (E, W, labels as the op read them, loss (1,), cos (N, C), lse (N,)) on E's device."""
    return aam_softmax_sc(E, W, labels, margin, scale)[:6]


def aam_softmax_backward(E, W, labels, cos, lse, margin, scale, grad_loss):
    """dsk_aam_softmax_bwd: (gE (N, D), gW (C, D)) = d loss / d (E, W) scaled by the device scalar ``grad_loss``."""
    return aam_softmax_sc_backward(E, W, labels, cos, lse, None, None, margin, scale, 1, 0, 0.0, grad_loss)


def subcentre_cosines(E, W, labels, subcentres):
    """dsk_aam_subcentre_cos: (N, K) fp32, each row's cosines to the K sub-centres of its own class (W is (C K, D),
    row c K + k sub-centre k of class c), in fp64 from the fp32 inputs and rounded once; NaN rows for labels outside
    [0, C).  These are the target cosines the sub-centre AAM-softmax forward takes its max over.

    Label cleaning and pruning after sub-centre training are torch plumbing on top (E a bank of embeddings, y its
    labels, W the trained (C K, D) weight)::

        sc = subcentre_cosines(E, W, y, K)                          # (N, K)
        best = sc.argmax(1)                                          # each utterance's nearest sub-centre
        counts = torch.zeros(C, K, dtype=torch.long, device=E.device)
        counts.index_put_((y, best), torch.ones_like(y), accumulate=True)
        dom = counts.argmax(1)                                       # (C,) each class's dominant sub-centre
        ang = torch.rad2deg(torch.acos(sc[torch.arange(len(y)), dom[y]].clamp(-1, 1)))
        keep = ang <= 75.0                                           # drop utterances far from their dominant centre
        W1 = W.view(C, K, -1)[torch.arange(C), dom]                  # (C, D) rows for a K = 1 fine-tune
    """
    K = subcentres
    C = aam_subcentre_args(W.shape[0] if W.dim() == 2 else 0, K, 0, 0.0)
    E, W, labels = _aam_inputs(E, W, labels)
    N, D = E.shape
    out = torch.empty(N, K, device=E.device, dtype=torch.float32)
    with torch.cuda.device(E.device):
        L.check(L.load().dsk_aam_subcentre_cos(E.data_ptr(), W.data_ptr(), labels.data_ptr(), N, C, K, D,
                                               out.data_ptr(), L.cur_stream()), "dsk_aam_subcentre_cos")
    return out


class AAMSoftmaxFn(torch.autograd.Function):
    """Additive angular margin softmax over a cosine classifier with K sub-centres per class and the inter-top-k
    penalty (K = 1, topk = 0: plain AAM-softmax); the loss is a device scalar."""

    @staticmethod
    def forward(ctx, E, W, labels, margin, scale, subcentres, topk, topk_margin):
        Ec, Wc, lab, loss, cos, lse, sub, top = aam_softmax_sc(E, W, labels, margin, scale, subcentres, topk,
                                                               topk_margin)
        ctx.save_for_backward(Ec, Wc, lab, cos, lse, sub, top)
        ctx.args = margin, scale, subcentres, topk, topk_margin
        return loss.reshape(())

    @staticmethod
    def backward(ctx, gl):
        E, W, lab, cos, lse, sub, top = ctx.saved_tensors
        gE, gW = aam_softmax_sc_backward(E, W, lab, cos, lse, sub, top, *ctx.args, gl)
        return ((gE if ctx.needs_input_grad[0] else None), (gW if ctx.needs_input_grad[1] else None)) + (None,) * 6


# ---- the class-sharded op (include/dsk.h, dsk_aam_shard_*): the stages of parallel.ShardedAAMSoftmaxLoss --------------
# Rank r holds the classes [c0, c1) of C, i.e. the rows [c0 K, c1 K) of the (C K, D) weight as W_r, and all N gathered
# rows.  Every tensor a stage returns is caller-owned; the handle's plan holds nothing between stages.

def _shard_tensor(t, name, shape, dtype, device):
    """A caller's tensor for a dsk_aam_shard_* call: on ``device``, of ``dtype`` and ``shape`` (None entries free) and
    contiguous, or RuntimeError (the C ABI sees pointers only)."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != device:
        raise RuntimeError(f"{name} must be a CUDA tensor on {device}")
    if t.dtype != dtype:
        raise RuntimeError(f"{name} must be {dtype}, got {t.dtype}")
    if t.dim() != len(shape) or any(s is not None and s != d for s, d in zip(shape, t.shape)):
        raise RuntimeError(f"{name} must have shape {tuple('*' if s is None else s for s in shape)}, got {tuple(t.shape)}")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be contiguous")
    return t


def _shard_rows(cos, labels, c0, c1):
    """The (N, c1 - c0) class cosines of a shard and the (N,) global labels; a valid range is the C ABI's check."""
    if not isinstance(cos, torch.Tensor) or cos.dim() != 2:
        raise RuntimeError("cos must be the (N, c1 - c0) shard cosines")
    dev, N = cos.device, cos.shape[0]
    _shard_tensor(cos, "cos", (N, c1 - c0), torch.float32, dev)
    _shard_tensor(labels, "labels", (N,), torch.int64, dev)
    return N, dev


def aam_shard_cos(E, W, labels, C, c0, c1, subcentres, topk):
    """dsk_aam_shard_cos: (cos (N, c1 - c0), sub (N, c1 - c0) uint8 or None when subcentres = 1, keys (N, topk) int64
    (the uint64 candidate keys' bits) or None when topk = 0)."""
    if not isinstance(E, torch.Tensor) or E.dim() != 2:
        raise RuntimeError("E must be the (N, D) gathered embeddings")
    N, D = E.shape
    dev, Cr = E.device, c1 - c0
    _shard_tensor(E, "E", (N, D), torch.float32, dev)
    _shard_tensor(W, "W", (Cr * subcentres, D), torch.float32, dev)
    _shard_tensor(labels, "labels", (N,), torch.int64, dev)
    cos = torch.empty(N, Cr, device=dev, dtype=torch.float32)
    sub = torch.empty(N, Cr, device=dev, dtype=torch.uint8) if subcentres > 1 else None
    keys = torch.empty(N, topk, device=dev, dtype=torch.int64) if topk > 0 else None
    with torch.cuda.device(dev):
        L.check(L.load().dsk_aam_shard_cos(_allpairs_handle(dev), E.data_ptr(), W.data_ptr(), labels.data_ptr(), N, C,
                                           c0, c1, subcentres, D, topk, cos.data_ptr(), L.ptr(sub), L.ptr(keys),
                                           L.cur_stream()), "dsk_aam_shard_cos")
    return cos, sub, keys


def aam_shard_merge(cos, labels, keys_all, R, C, c0, c1, topk, margin, scale, topk_margin):
    """dsk_aam_shard_merge: (top (N, topk) int32 or None, thr (N,) int64 (uint64 bits) or None, mloc (N,)) from the
    gathered candidate keys keys_all (R N topk,) in rank order."""
    N, dev = _shard_rows(cos, labels, c0, c1)
    if topk > 0:
        _shard_tensor(keys_all, "keys_all", (R * N * topk,) if keys_all.dim() == 1 else (R * N, topk), torch.int64,
                      dev)
    top = torch.empty(N, topk, device=dev, dtype=torch.int32) if topk > 0 else None
    thr = torch.empty(N, device=dev, dtype=torch.int64) if topk > 0 else None
    mloc = torch.empty(N, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        L.check(L.load().dsk_aam_shard_merge(cos.data_ptr(), labels.data_ptr(), L.ptr(keys_all), R, N, C, c0, c1, topk,
                                             float(margin), float(scale), float(topk_margin), L.ptr(top), L.ptr(thr),
                                             mloc.data_ptr(), L.cur_stream()), "dsk_aam_shard_merge")
    return top, thr, mloc


def aam_shard_partials(cos, labels, thr, maxima, R, C, c0, c1, topk, nb, margin, scale, topk_margin):
    """dsk_aam_shard_partials: (m (N,) the global row max, rec (N, 2 nb + 2) fp32 records) from the gathered maxima
    (R N,) in rank order."""
    N, dev = _shard_rows(cos, labels, c0, c1)
    if topk > 0:
        _shard_tensor(thr, "thr", (N,), torch.int64, dev)
    _shard_tensor(maxima, "maxima", (R * N,), torch.float32, dev)
    m = torch.empty(N, device=dev, dtype=torch.float32)
    rec = torch.empty(N, 2 * nb + 2, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        L.check(L.load().dsk_aam_shard_partials(cos.data_ptr(), labels.data_ptr(), L.ptr(thr), maxima.data_ptr(), R, N,
                                                C, c0, c1, topk, nb, float(margin), float(scale), float(topk_margin),
                                                m.data_ptr(), rec.data_ptr(), L.cur_stream()), "dsk_aam_shard_partials")
    return m, rec


def aam_shard_finish(rec_all, m, labels, R, C, nb):
    """dsk_aam_shard_finish: (loss (1,), lse (N,), row_loss (N,), den (N, 2)) from the gathered records
    (R N (2 nb + 2),) in rank order; the same bits on every rank and for every split."""
    if not isinstance(m, torch.Tensor) or m.dim() != 1:
        raise RuntimeError("m must be the (N,) row maxima")
    N, dev = m.shape[0], m.device
    _shard_tensor(m, "m", (N,), torch.float32, dev)
    _shard_tensor(labels, "labels", (N,), torch.int64, dev)
    _shard_tensor(rec_all, "rec_all", (R * N * (2 * nb + 2),) if rec_all.dim() == 1 else (R * N, 2 * nb + 2),
                  torch.float32, dev)
    loss = torch.empty(1, device=dev, dtype=torch.float32)
    lse, row_loss = (torch.empty(N, device=dev, dtype=torch.float32) for _ in range(2))
    den = torch.empty(N, 2, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        L.check(L.load().dsk_aam_shard_finish(rec_all.data_ptr(), m.data_ptr(), labels.data_ptr(), R, N, C, nb,
                                              loss.data_ptr(), lse.data_ptr(), row_loss.data_ptr(), den.data_ptr(),
                                              L.cur_stream()), "dsk_aam_shard_finish")
    return loss, lse, row_loss, den


def aam_shard_backward(E, W, labels, cos, sub, thr, m, den, C, c0, c1, margin, scale, subcentres, topk, topk_margin,
                       grad_loss):
    """dsk_aam_shard_bwd: (gW (shard rows, D), gE_part (N, D)): the shard's weight gradient and its partial gradient
    w.r.t. the normalised rows, scaled by the device scalar ``grad_loss``."""
    N, dev = _shard_rows(cos, labels, c0, c1)
    D = E.shape[1] if isinstance(E, torch.Tensor) and E.dim() == 2 else 0
    _shard_tensor(E, "E", (N, D), torch.float32, dev)
    _shard_tensor(W, "W", ((c1 - c0) * subcentres, D), torch.float32, dev)
    if subcentres > 1:
        _shard_tensor(sub, "sub", (N, c1 - c0), torch.uint8, dev)
    if topk > 0:
        _shard_tensor(thr, "thr", (N,), torch.int64, dev)
    _shard_tensor(m, "m", (N,), torch.float32, dev)
    _shard_tensor(den, "den", (N, 2), torch.float32, dev)
    gl = grad_loss.float().reshape(1).contiguous()
    gW, part = torch.empty_like(W), torch.empty_like(E)
    with torch.cuda.device(E.device):
        L.check(L.load().dsk_aam_shard_bwd(_allpairs_handle(E.device), E.data_ptr(), W.data_ptr(), labels.data_ptr(),
                                           cos.data_ptr(), L.ptr(sub), L.ptr(thr), m.data_ptr(), den.data_ptr(), N, C,
                                           c0, c1, subcentres, D, float(margin), float(scale), topk, float(topk_margin),
                                           gl.data_ptr(), gW.data_ptr(), part.data_ptr(), L.cur_stream()),
                "dsk_aam_shard_bwd")
    return gW, part


def aam_shard_backward_rows(E_local, parts, R):
    """dsk_aam_shard_bwd_rows: gE (n, D) of this rank's rows from the R ranks' partials of them (R n D,), rank order."""
    if not isinstance(E_local, torch.Tensor) or E_local.dim() != 2:
        raise RuntimeError("E_local must be this rank's (n, D) embeddings")
    n, D = E_local.shape
    _shard_tensor(E_local, "E_local", (n, D), torch.float32, E_local.device)
    _shard_tensor(parts, "parts", (R * n * D,) if parts.dim() == 1 else (R * n, D), torch.float32, E_local.device)
    gE = torch.empty_like(E_local)
    with torch.cuda.device(E_local.device):
        L.check(L.load().dsk_aam_shard_bwd_rows(E_local.data_ptr(), parts.data_ptr(), R, n, D, gE.data_ptr(),
                                                L.cur_stream()), "dsk_aam_shard_bwd_rows")
    return gE


# ---------------------------------------------------------------------------------------------------
# generalised end-to-end (GE2E) loss
# ---------------------------------------------------------------------------------------------------
GE2E_METHODS = {"softmax": L.DSK_GE2E_SOFTMAX, "contrast": L.DSK_GE2E_CONTRAST}


def _ge2e_method(method):
    if method not in GE2E_METHODS:
        raise ValueError(f"GE2E method must be one of {sorted(GE2E_METHODS)}, got {method!r}")
    return GE2E_METHODS[method]


def ge2e(E, csr, V, w, b, method):
    """dsk_ge2e: (E as the op read it, loss (1,), cos (N, P), rec (N,)) on E's device.  ``csr`` = (order, offsets, col)
    int64 device tensors (``model.ge2e_batch``), ``V`` the number of valid rows, ``w`` / ``b`` fp32 device scalars."""
    m = _ge2e_method(method)
    if not E.is_cuda:
        raise RuntimeError("the GE2E loss needs CUDA tensors; there is no CPU fallback")
    if E.dim() != 2:
        raise RuntimeError(f"expected embeddings (N, D), got {tuple(E.shape)}")
    E = E.detach().float().contiguous()
    order, offsets, col = csr
    (N, D), P = E.shape, offsets.numel() - 1
    if order.numel() != N or col.numel() != N:
        raise RuntimeError(f"GE2E: {order.numel()} labels for {N} embeddings")
    dev = E.device
    for t in (order, offsets, col, w, b):
        if t.device != dev:
            raise RuntimeError("GE2E: embeddings, speaker lists and the scalars w, b must be on one device")
    loss = torch.empty(1, device=dev, dtype=torch.float32)
    cos = torch.empty(N, P, device=dev, dtype=torch.float32)
    rec = torch.empty(N, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        L.check(L.load().dsk_ge2e(_allpairs_handle(dev), E.data_ptr(), N, D, order.data_ptr(), offsets.data_ptr(),
                                  col.data_ptr(), P, int(V), w.data_ptr(), b.data_ptr(), m, loss.data_ptr(),
                                  cos.data_ptr(), rec.data_ptr(), L.cur_stream()), "dsk_ge2e")
    return E, loss, cos, rec


def ge2e_backward(E, csr, V, w, b, method, cos, rec, grad_loss):
    """dsk_ge2e_bwd: (gE (N, D), gw (), gb ()) = d loss / d (E, w, b) scaled by the device scalar ``grad_loss``; gb is
    exactly 0 for ``softmax``."""
    order, offsets, col = csr
    (N, D), P = E.shape, offsets.numel() - 1
    gl = grad_loss.float().reshape(1).contiguous()
    gE = torch.empty_like(E)
    gw = torch.empty((), device=E.device, dtype=torch.float32)
    gb = torch.empty((), device=E.device, dtype=torch.float32)
    with torch.cuda.device(E.device):
        L.check(L.load().dsk_ge2e_bwd(_allpairs_handle(E.device), E.data_ptr(), N, D, order.data_ptr(),
                                      offsets.data_ptr(), col.data_ptr(), P, int(V), w.data_ptr(), b.data_ptr(),
                                      _ge2e_method(method), cos.data_ptr(), rec.data_ptr(), gl.data_ptr(), gE.data_ptr(),
                                      gw.data_ptr(), gb.data_ptr(), L.cur_stream()), "dsk_ge2e_bwd")
    return gE, gw, gb


def ge2e_rows(E, csr, V, w, b, method, row0, rows):
    """dsk_ge2e_rows: rows [row0, row0 + rows) of ``ge2e`` on the whole batch E (N, D) -> (E fp32 contiguous, cos
    (rows, P), rec (rows,), row_loss (rows,)), the same bits as those rows of ``ge2e``.  ``csr`` is the whole batch's.
    The plan is cached per (N, P, D, row0, rows)."""
    m = _ge2e_method(method)
    if not E.is_cuda or E.dim() != 2:
        raise RuntimeError(f"GE2E: expected CUDA embeddings (N, D), got {tuple(E.shape)} on {E.device}")
    E = E.detach().float().contiguous()
    order, offsets, col = csr
    (N, D), P, dev, n = E.shape, offsets.numel() - 1, E.device, max(int(rows), 0)
    if order.numel() != N or col.numel() != N:
        raise RuntimeError(f"GE2E: {order.numel()} labels for {N} embeddings")
    for t in (order, offsets, col, w, b):
        if t.device != dev:
            raise RuntimeError("GE2E: embeddings, speaker lists and the scalars w, b must be on one device")
    cos = torch.empty(n, P, device=dev, dtype=torch.float32)
    rec, row_loss = (torch.empty(n, device=dev, dtype=torch.float32) for _ in range(2))
    with torch.cuda.device(dev):
        L.check(L.load().dsk_ge2e_rows(_allpairs_handle(dev), E.data_ptr(), N, D, order.data_ptr(), offsets.data_ptr(),
                                       col.data_ptr(), P, int(V), w.data_ptr(), b.data_ptr(), m, int(row0), int(rows),
                                       cos.data_ptr(), rec.data_ptr(), row_loss.data_ptr(), L.cur_stream()),
                "dsk_ge2e_rows")
    return E, cos, rec, row_loss


def ge2e_mean(row_loss, V):
    """dsk_ge2e_mean: loss (1,) from the row losses (N,) of the whole batch, the bits of ``ge2e``'s loss."""
    loss = torch.empty(1, device=row_loss.device, dtype=torch.float32)
    with torch.cuda.device(row_loss.device):
        L.check(L.load().dsk_ge2e_mean(row_loss.data_ptr(), row_loss.numel(), int(V), loss.data_ptr(), L.cur_stream()),
                "dsk_ge2e_mean")
    return loss


def ge2e_dcos_rows(cos, rec, csr, V, w, b, method, row0, rows, grad_loss):
    """dsk_ge2e_dcos_rows: from the range's ``ge2e_rows`` outputs -> (dcos (rows, P) with the target column zeroed, tdc
    (rows,) the target column's dcos, gw (), gb ()): the range's part of ``ge2e_backward`` and its shares of gw, gb."""
    _, offsets, col = csr
    n, P = max(int(rows), 0), offsets.numel() - 1
    dev = cos.device
    if tuple(cos.shape) != (n, P) or tuple(rec.shape) != (n,):
        raise RuntimeError(f"GE2E: expected cos ({n}, {P}) and rec ({n},) of the row range, got {tuple(cos.shape)} "
                           f"and {tuple(rec.shape)}")
    for t in (cos, rec, offsets, col, w, b):
        if not t.is_cuda or t.device != dev:
            raise RuntimeError("GE2E: cos, rec, speaker lists and the scalars w, b must be on one CUDA device")
    cos, rec = cos.float().contiguous(), rec.float().contiguous()
    gl = grad_loss.float().reshape(1).contiguous()
    dcos = torch.empty(n, P, device=dev, dtype=torch.float32)
    tdc = torch.empty(n, device=dev, dtype=torch.float32)
    gw, gb = (torch.empty((), device=dev, dtype=torch.float32) for _ in range(2))
    with torch.cuda.device(dev):
        L.check(L.load().dsk_ge2e_dcos_rows(cos.data_ptr(), rec.data_ptr(), col.numel(), offsets.data_ptr(),
                                            col.data_ptr(), P, int(V), w.data_ptr(), b.data_ptr(), _ge2e_method(method),
                                            gl.data_ptr(), int(row0), int(rows), dcos.data_ptr(), tdc.data_ptr(),
                                            gw.data_ptr(), gb.data_ptr(), L.cur_stream()), "dsk_ge2e_dcos_rows")
    return dcos, tdc, gw, gb


def ge2e_backward_rows(E, csr, dcos, tdc, row0, rows):
    """dsk_ge2e_bwd_rows: rows [row0, row0 + rows) of ``ge2e_backward``'s gE -> (rows, D), the same bits.  ``dcos``
    (N, P) and ``tdc`` (N,) are every range's ``ge2e_dcos_rows`` outputs, concatenated in row order."""
    order, offsets, col = csr
    (N, D), P = E.shape, offsets.numel() - 1
    if dcos.shape != (N, P) or tdc.shape != (N,):
        raise RuntimeError(f"GE2E: expected dcos ({N}, {P}) and tdc ({N},), got {tuple(dcos.shape)} and "
                           f"{tuple(tdc.shape)}")
    if not E.is_cuda or any(t.device != E.device for t in (order, offsets, col, dcos, tdc)):
        raise RuntimeError("GE2E: embeddings, speaker lists, dcos and tdc must be on one CUDA device")
    E = E.detach().float().contiguous()
    dcos, tdc = dcos.float().contiguous(), tdc.float().contiguous()
    gE = torch.empty(max(int(rows), 0), D, device=E.device, dtype=torch.float32)
    with torch.cuda.device(E.device):
        L.check(L.load().dsk_ge2e_bwd_rows(_allpairs_handle(E.device), E.data_ptr(), N, D, order.data_ptr(),
                                           offsets.data_ptr(), col.data_ptr(), P, dcos.data_ptr(), tdc.data_ptr(),
                                           int(row0), int(rows), gE.data_ptr(), L.cur_stream()), "dsk_ge2e_bwd_rows")
    return gE


class GE2EFn(torch.autograd.Function):
    """GE2E loss over (E, w, b) against the batch's speaker centroids; the loss is a device scalar.  ``csr`` and ``V``
    as in ``ge2e``."""

    @staticmethod
    def forward(ctx, E, w, b, csr, V, method):
        wc, bc = (t.detach().float().reshape(1).contiguous() for t in (w, b))
        Ec, loss, cos, rec = ge2e(E, csr, V, wc, bc, method)
        ctx.save_for_backward(Ec, wc, bc, cos, rec, *csr)
        ctx.V, ctx.method, ctx.shapes = V, method, (w.shape, b.shape)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, gl):
        E, w, b, cos, rec, order, offsets, col = ctx.saved_tensors
        gE, gw, gb = ge2e_backward(E, (order, offsets, col), ctx.V, w, b, ctx.method, cos, rec, gl)
        ni = ctx.needs_input_grad
        return (gE if ni[0] else None, gw.reshape(ctx.shapes[0]) if ni[1] else None,
                gb.reshape(ctx.shapes[1]) if ni[2] else None, None, None, None)


# ---------------------------------------------------------------------------------------------------
# supervised-contrastive loss (NT-Xent with one label per utterance)
# ---------------------------------------------------------------------------------------------------
def _labels_on(labels, N, dev):
    labels = torch.as_tensor(labels)
    if labels.dtype.is_floating_point or labels.dtype == torch.bool:
        raise ValueError(f"supervised-contrastive labels must be integers, got {labels.dtype}")
    if labels.shape != (N,):
        raise RuntimeError(f"expected labels of shape ({N},), got {tuple(labels.shape)}")
    if not labels.is_cuda:   # a pageable copy would wait for the stream; a pinned one is queued like a kernel
        return labels.to(torch.int64).contiguous().pin_memory().to(dev, non_blocking=True)
    return labels.to(device=dev, dtype=torch.int64).contiguous()


def supcon(E, labels, V, tau):
    """dsk_supcon: (E, labels as the op read them, loss (1,), cos (N, N), lse (N,)) on E's device.  ``V`` is the number
    of valid rows (``model.supcon_valid_count`` of the labels), ``tau`` the temperature."""
    if not E.is_cuda:
        raise RuntimeError("the supervised-contrastive loss needs CUDA tensors; there is no CPU fallback")
    if E.dim() != 2:
        raise RuntimeError(f"expected embeddings (N, D), got {tuple(E.shape)}")
    E = E.detach().float().contiguous()
    N, D = E.shape
    dev = E.device
    labels = _labels_on(labels, N, dev)
    loss = torch.empty(1, device=dev, dtype=torch.float32)
    cos = torch.empty(N, N, device=dev, dtype=torch.float32)
    lse = torch.empty(N, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        L.check(L.load().dsk_supcon(_allpairs_handle(dev), E.data_ptr(), labels.data_ptr(), N, D, int(V), float(tau),
                                    loss.data_ptr(), cos.data_ptr(), lse.data_ptr(), L.cur_stream()), "dsk_supcon")
    return E, labels, loss, cos, lse


def supcon_backward(E, labels, V, tau, cos, lse, grad_loss):
    """dsk_supcon_bwd: gE (N, D) = d loss / d E scaled by the device scalar ``grad_loss``, from the forward's cos and
    lse."""
    N, D = E.shape
    gl = grad_loss.float().reshape(1).contiguous()
    gE = torch.empty_like(E)
    with torch.cuda.device(E.device):
        L.check(L.load().dsk_supcon_bwd(_allpairs_handle(E.device), E.data_ptr(), labels.data_ptr(), cos.data_ptr(),
                                        lse.data_ptr(), N, D, int(V), float(tau), gl.data_ptr(), gE.data_ptr(),
                                        L.cur_stream()), "dsk_supcon_bwd")
    return gE


class SupConFn(torch.autograd.Function):
    """Supervised-contrastive loss over the batch's cosine matrix; the loss is a device scalar.  ``V`` and ``tau`` as in
    ``supcon``."""

    @staticmethod
    def forward(ctx, E, labels, V, tau):
        Ec, lab, loss, cos, lse = supcon(E, labels, V, tau)
        ctx.save_for_backward(Ec, lab, cos, lse)
        ctx.V, ctx.tau = V, tau
        return loss.reshape(())

    @staticmethod
    def backward(ctx, gl):
        E, lab, cos, lse = ctx.saved_tensors
        return supcon_backward(E, lab, ctx.V, ctx.tau, cos, lse, gl), None, None, None


# ---------------------------------------------------------------------------------------------------
# cosine scoring and cohort statistics (AS-norm)
# ---------------------------------------------------------------------------------------------------
def _score_rows(X, what):
    if not X.is_cuda:
        raise RuntimeError(f"{what} needs CUDA tensors; there is no CPU fallback")
    if X.dim() != 2:
        raise RuntimeError(f"{what}: expected a 2-D (rows, D) tensor, got shape {tuple(X.shape)}")
    return X.detach().float().contiguous()


def _score_pair(A, B, what):
    A, B = _score_rows(A, what), _score_rows(B, what)
    if A.shape[1] != B.shape[1]:
        raise RuntimeError(f"{what}: embedding sizes differ ({A.shape[1]} and {B.shape[1]})")
    if A.device != B.device:
        raise RuntimeError(f"{what}: both tensors must be on one device")
    return A, B


def cosine_matrix(A, B):
    """dsk_cosine_matrix: cos (M, Nc) fp32 = normalised rows of A (M, D) times those of B (Nc, D)."""
    A, B = _score_pair(A, B, "cosine_matrix")
    (M, D), Nc = A.shape, B.shape[0]
    cos = torch.empty(M, Nc, device=A.device, dtype=torch.float32)
    with torch.cuda.device(A.device):
        L.check(L.load().dsk_cosine_matrix(_allpairs_handle(A.device), A.data_ptr(), M, B.data_ptr(), Nc, D,
                                           cos.data_ptr(), L.cur_stream()), "dsk_cosine_matrix")
    return cos


def topk_mean_std(S, k):
    """dsk_topk_mean_std: (mean, std) (rows,) of the k largest values of every row of S (rows, cols) (its row stride is
    kept: a column slice of a row-major matrix needs no copy)."""
    if not S.is_cuda:
        raise RuntimeError("topk_mean_std needs CUDA tensors; there is no CPU fallback")
    if S.dim() != 2 or S.dtype != torch.float32 or S.stride(1) != 1:
        raise RuntimeError(f"topk_mean_std: expected a row-major fp32 (rows, cols) tensor, got {S.dtype} {tuple(S.shape)}")
    rows, cols = S.shape
    mean = torch.empty(rows, device=S.device, dtype=torch.float32)
    std = torch.empty_like(mean)
    with torch.cuda.device(S.device):
        L.check(L.load().dsk_topk_mean_std(S.data_ptr(), rows, cols, S.stride(0), int(k), mean.data_ptr(),
                                           std.data_ptr(), L.cur_stream()), "dsk_topk_mean_std")
    return mean, std


def cohort_stats(E, cohort, k):
    """dsk_cohort_stats: (mean, std) (M,) of the k largest cosines of every row of E against the cohort."""
    E, C = _score_pair(E, cohort, "cohort_stats")
    (M, D), Nc = E.shape, C.shape[0]
    mean = torch.empty(M, device=E.device, dtype=torch.float32)
    std = torch.empty_like(mean)
    with torch.cuda.device(E.device):
        L.check(L.load().dsk_cohort_stats(_allpairs_handle(E.device), E.data_ptr(), M, C.data_ptr(), Nc, D, int(k),
                                          mean.data_ptr(), std.data_ptr(), L.cur_stream()), "dsk_cohort_stats")
    return mean, std


def score_trials(X, trials, mean=None, std=None):
    """dsk_score_trials: (raw (T,), normed (T,) or None) for trials (T, 2) of row indices into X (U, D); ``mean`` /
    ``std`` (U,) are the rows' cohort statistics (AS-norm), or None for raw scores only."""
    X = _score_rows(X, "score_trials")
    trials = torch.as_tensor(trials)
    if trials.dim() != 2 or trials.shape[1] != 2 or trials.shape[0] < 1:
        raise RuntimeError(f"score_trials: expected trials of shape (T, 2) with T >= 1, got {tuple(trials.shape)}")
    trials = trials.to(device=X.device, dtype=torch.int64).contiguous()
    (U, D), T = X.shape, trials.shape[0]
    if (mean is None) != (std is None):
        raise RuntimeError("score_trials: give both mean and std, or neither")
    if mean is not None:
        mean, std = (t.detach().to(device=X.device, dtype=torch.float32).contiguous() for t in (mean, std))
        if mean.shape != (U,) or std.shape != (U,):
            raise RuntimeError(f"score_trials: expected mean and std of shape ({U},)")
    raw = torch.empty(T, device=X.device, dtype=torch.float32)
    normed = None if mean is None else torch.empty_like(raw)
    with torch.cuda.device(X.device):
        L.check(L.load().dsk_score_trials(X.data_ptr(), U, D, trials.data_ptr(), T, L.ptr(mean), L.ptr(std),
                                          raw.data_ptr(), L.ptr(normed), L.cur_stream()), "dsk_score_trials")
    return raw, normed


# ---------------------------------------------------------------------------------------------------
# identification: exact top-k search, class centroids
# ---------------------------------------------------------------------------------------------------
def topk_indices(S, k):
    """dsk_topk_indices: (idx int64 (rows, k), val fp32 (rows, k)) of the k first columns of every row of S (rows, cols)
    in the search order (descending, ties to the lower column, -0 == +0, NaN last); the row stride is kept."""
    if not S.is_cuda:
        raise RuntimeError("topk_indices needs CUDA tensors; there is no CPU fallback")
    if S.dim() != 2 or S.dtype != torch.float32 or S.stride(1) != 1:
        raise RuntimeError(f"topk_indices: expected a row-major fp32 (rows, cols) tensor, got {S.dtype} {tuple(S.shape)}")
    rows, cols = S.shape
    k = int(k)
    idx = torch.empty(rows, max(k, 0), device=S.device, dtype=torch.int64)
    val = torch.empty(rows, max(k, 0), device=S.device, dtype=torch.float32)
    with torch.cuda.device(S.device):
        L.check(L.load().dsk_topk_indices(S.data_ptr(), rows, cols, S.stride(0), k, idx.data_ptr(), val.data_ptr(),
                                          L.cur_stream()), "dsk_topk_indices")
    return idx, val


def cosine_topk(Q, G, k):
    """dsk_cosine_topk: (idx int64 (M, k), val fp32 (M, k)) of the k largest cosines of every row of Q (M, D) against
    the gallery G (Ng, D), any Ng >= k, in the search order; val is the cosine cosine_matrix gives for the pair."""
    Q, G = _score_pair(Q, G, "cosine_topk")
    (M, D), Ng, k = Q.shape, G.shape[0], int(k)
    idx = torch.empty(M, max(k, 0), device=Q.device, dtype=torch.int64)
    val = torch.empty(M, max(k, 0), device=Q.device, dtype=torch.float32)
    with torch.cuda.device(Q.device):
        L.check(L.load().dsk_cosine_topk(_allpairs_handle(Q.device), Q.data_ptr(), M, G.data_ptr(), Ng, D, k,
                                         idx.data_ptr(), val.data_ptr(), L.cur_stream()), "dsk_cosine_topk")
    return idx, val


def class_centroids(X, order, offsets):
    """dsk_class_centroids: (S, D) fp32 mean of the normalised rows X[order[offsets[s]:offsets[s+1]]] per class s, in
    fp64 in that order; ``order`` / ``offsets`` (S + 1,) are int64 (a CSR of the classes' rows)."""
    X = _score_rows(X, "class_centroids")
    order = torch.as_tensor(order).to(device=X.device, dtype=torch.int64).contiguous()
    offsets = torch.as_tensor(offsets).to(device=X.device, dtype=torch.int64).contiguous()
    if order.dim() != 1 or offsets.dim() != 1 or offsets.numel() < 2:
        raise RuntimeError(f"class_centroids: expected 1-D order and offsets with >= 2 entries, got "
                           f"{tuple(order.shape)} and {tuple(offsets.shape)}")
    (U, D), S = X.shape, offsets.numel() - 1
    out = torch.empty(S, D, device=X.device, dtype=torch.float32)
    with torch.cuda.device(X.device):
        L.check(L.load().dsk_class_centroids(X.data_ptr(), U, D, order.data_ptr(), offsets.data_ptr(), S,
                                             out.data_ptr(), L.cur_stream()), "dsk_class_centroids")
    return out


# ---------------------------------------------------------------------------------------------------
# diarization: agglomerative clustering
# ---------------------------------------------------------------------------------------------------
LINKAGES = {"average": L.DSK_LINKAGE_AVERAGE, "complete": L.DSK_LINKAGE_COMPLETE}


def ahc(S, linkage="average", num_clusters=None, threshold=None, return_rounds=False):
    """dsk_ahc: agglomerative clustering of N items from their similarities S (N, N) fp32 on the device (higher =
    closer, e.g. ``cosine_matrix(E, E)``; only the strict upper triangle is read, the row stride is kept), on the
    distance 1 - S in fp64.  -> (Z np.float64 (m, 4) in scipy's linkage format, labels torch.int32 (N,) on S's device,
    the flat clusters numbered by their smallest member).  ``num_clusters``: stop at that many clusters (exact: the cut
    of the full tree).  ``threshold``: merge only at heights <= threshold (a distance).  Neither: the full tree, m =
    N - 1.  ``return_rounds`` adds the number of merge rounds.  RuntimeError on a non-finite similarity."""
    if linkage not in LINKAGES:
        raise ValueError(f"ahc: linkage must be one of {sorted(LINKAGES)}, got {linkage!r}")
    if num_clusters is not None and threshold is not None:
        raise ValueError("ahc: give num_clusters or threshold, not both")
    if not S.is_cuda:
        raise RuntimeError("ahc needs a CUDA tensor; there is no CPU fallback")
    if S.dim() != 2 or S.shape[0] != S.shape[1] or S.dtype != torch.float32 or S.stride(1) != 1:
        raise RuntimeError(f"ahc: expected a row-major fp32 (N, N) tensor, got {S.dtype} {tuple(S.shape)}")
    N = S.shape[0]
    stop_k = 1 if num_clusters is None else int(num_clusters)
    stop_h = float("inf") if threshold is None else float(threshold)
    Z = np.empty((max(N - 1, 1), 4), np.float64)
    labels = np.empty(max(N, 1), np.int32)
    m, rounds = ctypes.c_int32(0), ctypes.c_int32(0)
    with torch.cuda.device(S.device):
        L.check(L.load().dsk_ahc(S.data_ptr(), N, S.stride(0), LINKAGES[linkage], stop_k, stop_h,
                                 Z.ctypes.data_as(ctypes.c_void_p), ctypes.byref(m),
                                 labels.ctypes.data_as(ctypes.c_void_p), ctypes.byref(rounds), L.cur_stream()), "dsk_ahc")
    out = (Z[:m.value].copy(), torch.from_numpy(labels).to(S.device))
    return out + (rounds.value,) if return_rounds else out


def spectral_cluster(S, p_values, max_speakers=8, num_speakers=None, kmeans_iters=100, return_embedding=False):
    """dsk_spectral_cluster: spectral clustering of N items from their similarities S (N, N) fp32 on the device (higher
    = closer; both triangles are read, the diagonal never, the row stride is kept) with NME-SC speaker counting over
    the pruning levels ``p_values`` (strictly increasing in [1, N - 1]).  ``num_speakers``: None estimates the count
    (at most ``max_speakers``), an int fixes it.  -> (labels torch.int32 (N,) on S's device numbered by each cluster's
    smallest member, k, p_index into p_values, eigenvalues np.float64 (n_p, m), lambda_max (n_p,), ratio (n_p,)), plus
    the (N, m - 1) fp64 device embedding (its first k columns the eigenvectors) with ``return_embedding``.
    RuntimeError on a non-finite off-diagonal similarity or on bad arguments."""
    if not S.is_cuda:
        raise RuntimeError("spectral_cluster needs a CUDA tensor; there is no CPU fallback")
    if S.dim() != 2 or S.shape[0] != S.shape[1] or S.dtype != torch.float32 or S.stride(1) != 1:
        raise RuntimeError(f"spectral_cluster: expected a row-major fp32 (N, N) tensor, got {S.dtype} {tuple(S.shape)}")
    N = S.shape[0]
    pv = np.ascontiguousarray(np.asarray(p_values, np.int64).reshape(-1).astype(np.int32))
    ns = 0 if num_speakers is None else int(num_speakers)
    m = ns + 1 if ns else min(int(max_speakers) + 1, max(N, 1))
    labels = np.empty(max(N, 1), np.int32)
    eig = np.empty((max(pv.size, 1), max(m, 1)), np.float64)
    lmax = np.empty(max(pv.size, 1), np.float64)
    ratio = np.empty(max(pv.size, 1), np.float64)
    k, t = ctypes.c_int32(0), ctypes.c_int32(0)
    emb = torch.zeros((max(N, 1), max(m - 1, 1)), dtype=torch.float64, device=S.device) if return_embedding else None

    def host(a):
        return a.ctypes.data_as(ctypes.c_void_p)

    with torch.cuda.device(S.device):
        L.check(L.load().dsk_spectral_cluster(S.data_ptr(), N, S.stride(0), host(pv), pv.size, int(max_speakers), ns,
                                              int(kmeans_iters), host(labels), ctypes.byref(k), ctypes.byref(t),
                                              host(eig), host(lmax), host(ratio),
                                              emb.data_ptr() if emb is not None else None, L.cur_stream()),
                "dsk_spectral_cluster")
    out = (torch.from_numpy(labels).to(S.device), k.value, t.value, eig, lmax, ratio)
    return out + (emb,) if return_embedding else out


# ---------------------------------------------------------------------------------------------------
# PLDA backend: fp64 fit statistics, transforms, LLR scoring
# ---------------------------------------------------------------------------------------------------
NORM_MODES = {"none": L.DSK_NORM_NONE, "length": L.DSK_NORM_LENGTH, "plda": L.DSK_NORM_PLDA}


def _f64_vec(v, device, n, what):
    if v is None:
        return None
    v = torch.as_tensor(v).detach().to(device=device, dtype=torch.float64).contiguous()
    if v.shape != (n,):
        raise RuntimeError(f"{what}: expected shape ({n},), got {tuple(v.shape)}")
    return v


def _counts(counts, device, n, what):
    if counts is None:
        return None
    c = torch.as_tensor(counts).detach().to(device=device, dtype=torch.int32).contiguous()
    if c.shape != (n,):
        raise RuntimeError(f"{what}: expected counts of shape ({n},), got {tuple(c.shape)}")
    return c


def class_sums_f64(X, order, offsets, mu=None):
    """dsk_class_sums_f64: (C, D) fp64 sums of X[u] - mu over u = order[offsets[c]:offsets[c+1]] per class c, in that
    order; ``mu`` (D,) fp64 or None (0)."""
    X = _score_rows(X, "class_sums_f64")
    order = torch.as_tensor(order).to(device=X.device, dtype=torch.int64).contiguous()
    offsets = torch.as_tensor(offsets).to(device=X.device, dtype=torch.int64).contiguous()
    if order.dim() != 1 or offsets.dim() != 1 or offsets.numel() < 2:
        raise RuntimeError(f"class_sums_f64: expected 1-D order and offsets with >= 2 entries, got "
                           f"{tuple(order.shape)} and {tuple(offsets.shape)}")
    (N, D), C = X.shape, offsets.numel() - 1
    mu = _f64_vec(mu, X.device, D, "class_sums_f64")
    out = torch.empty(C, D, device=X.device, dtype=torch.float64)
    with torch.cuda.device(X.device):
        L.check(L.load().dsk_class_sums_f64(X.data_ptr(), N, D, order.data_ptr(), offsets.data_ptr(), C, L.ptr(mu),
                                            out.data_ptr(), L.cur_stream()), "dsk_class_sums_f64")
    return out


def gram_f64(X, mu=None):
    """dsk_gram_f64: (D, D) fp64 sum over the rows of (X[u] - mu)(X[u] - mu)^T on the fp64 tensor cores, exactly
    symmetric and the same bits on every call; ``mu`` (D,) fp64 or None (0)."""
    X = _score_rows(X, "gram_f64")
    N, D = X.shape
    mu = _f64_vec(mu, X.device, D, "gram_f64")
    G = torch.empty(D, D, device=X.device, dtype=torch.float64)
    with torch.cuda.device(X.device):
        L.check(L.load().dsk_gram_f64(X.data_ptr(), N, D, L.ptr(mu), G.data_ptr(), L.cur_stream()), "dsk_gram_f64")
    return G


def affine_norm_f64(X, A, c=None, mode="none", psi=None, counts=None):
    """dsk_affine_norm_f64: (N, d) fp32 rows s_u A (X[u] - c), accumulated in fp64 and rounded once.  ``mode``: "none"
    (s = 1), "length" (s = sqrt(d) / ||A (x - c)||) or "plda" (s = sqrt(d / sum_l z_l^2 / (psi_l + 1 / n_u)), with
    ``counts`` (N,) the n_u, None for 1)."""
    if mode not in NORM_MODES:
        raise ValueError(f"affine_norm_f64: mode must be one of {sorted(NORM_MODES)}, got {mode!r}")
    X = _score_rows(X, "affine_norm_f64")
    N, D = X.shape
    A = torch.as_tensor(A).detach().to(device=X.device, dtype=torch.float64).contiguous()
    if A.dim() != 2 or A.shape[1] != D:
        raise RuntimeError(f"affine_norm_f64: expected A of shape (d, {D}), got {tuple(A.shape)}")
    d = A.shape[0]
    c = _f64_vec(c, X.device, D, "affine_norm_f64")
    psi = _f64_vec(psi, X.device, d, "affine_norm_f64")
    if mode == "plda" and psi is None:
        raise RuntimeError("affine_norm_f64: mode 'plda' needs psi")
    counts = _counts(counts, X.device, N, "affine_norm_f64")
    Y = torch.empty(N, d, device=X.device, dtype=torch.float32)
    with torch.cuda.device(X.device):
        L.check(L.load().dsk_affine_norm_f64(X.data_ptr(), N, D, A.data_ptr(), d, L.ptr(c), NORM_MODES[mode], L.ptr(psi),
                                             L.ptr(counts), Y.data_ptr(), L.cur_stream()), "dsk_affine_norm_f64")
    return Y


def plda_score_trials(Y, psi, trials, counts=None):
    """dsk_plda_score_trials: (T,) fp32 PLDA LLRs of trials (T, 2) (enrolment, test) of row indices into the
    transformed rows Y (U, d); ``counts`` (U,) the utterances averaged into each row (None: 1), used on the enrolment
    side.  An index outside [0, U) or a count < 1 gives NaN."""
    Y = _score_rows(Y, "plda_score_trials")
    U, d = Y.shape
    trials = torch.as_tensor(trials)
    if trials.dim() != 2 or trials.shape[1] != 2 or trials.shape[0] < 1:
        raise RuntimeError(f"plda_score_trials: expected trials of shape (T, 2) with T >= 1, got {tuple(trials.shape)}")
    trials = trials.to(device=Y.device, dtype=torch.int64).contiguous()
    psi = _f64_vec(psi, Y.device, d, "plda_score_trials")
    counts = _counts(counts, Y.device, U, "plda_score_trials")
    llr = torch.empty(trials.shape[0], device=Y.device, dtype=torch.float32)
    with torch.cuda.device(Y.device):
        L.check(L.load().dsk_plda_score_trials(Y.data_ptr(), U, d, psi.data_ptr(), L.ptr(counts), trials.data_ptr(),
                                               trials.shape[0], llr.data_ptr(), L.cur_stream()), "dsk_plda_score_trials")
    return llr


def plda_score_matrix(Ya, Yb, psi):
    """dsk_plda_score_matrix: (M, N) fp32 n = 1 PLDA LLRs of every row of Ya (M, d) against every row of Yb (N, d)."""
    Ya, Yb = _score_pair(Ya, Yb, "plda_score_matrix")
    (M, d), N = Ya.shape, Yb.shape[0]
    psi = _f64_vec(psi, Ya.device, d, "plda_score_matrix")
    S = torch.empty(M, N, device=Ya.device, dtype=torch.float32)
    with torch.cuda.device(Ya.device):
        L.check(L.load().dsk_plda_score_matrix(Ya.data_ptr(), M, Yb.data_ptr(), N, d, psi.data_ptr(), S.data_ptr(), N,
                                               L.cur_stream()), "dsk_plda_score_matrix")
    return S


# ---------------------------------------------------------------------------------------------------
# VBx: Bayesian HMM clustering of window embeddings in the PLDA space
# ---------------------------------------------------------------------------------------------------
def vbx(X, offsets, init_labels, phi, Fa, Fb, loop_p, init_smoothing, max_iters, epsilon):
    """dsk_vbx over the recordings offsets[r] .. offsets[r + 1] of the PLDA-space rows X (W, d) (CUDA; fp32 without
    the scoring normalisation), ``offsets`` (R + 1,) on the CPU, ``init_labels`` (W,) CUDA or CPU, ``phi`` (d,) the
    PLDA's psi.  S = min(1 + the largest label, DSK_VBX_MAX_SPEAKERS) columns; recording r has S_r = 1 + its largest
    label speakers, and a label outside [0, S) makes its recording NaN with labels -1.
    -> device tensors (gamma (W, S) fp64, pi (R, S) fp64, elbo (R, max_iters) fp64 (NaN past a recording's last
    iteration), iters (R,) int32, labels (W,) int32 (the argmax of each gamma row, not renumbered))."""
    X = _score_rows(X, "vbx")
    W, d = X.shape
    off = torch.as_tensor(offsets)
    if off.is_cuda:
        raise RuntimeError("vbx: offsets must be a CPU tensor or array")
    off = off.to(torch.int64).contiguous()
    if off.dim() != 1 or off.numel() < 2:
        raise RuntimeError(f"vbx: expected 1-D offsets with >= 2 entries, got shape {tuple(off.shape)}")
    lab = torch.as_tensor(init_labels).detach().to(device=X.device, dtype=torch.int32).contiguous()
    if lab.shape != (W,):
        raise RuntimeError(f"vbx: expected init_labels of shape ({W},), got {tuple(lab.shape)}")
    phi = _f64_vec(phi, X.device, d, "vbx")
    R = off.numel() - 1
    S = max(1, min(int(lab.max().item()) + 1, L.DSK_VBX_MAX_SPEAKERS)) if W else 1
    gamma = torch.empty(W, S, device=X.device, dtype=torch.float64)
    pi = torch.empty(R, S, device=X.device, dtype=torch.float64)
    elbo = torch.empty(R, max(int(max_iters), 1), device=X.device, dtype=torch.float64)
    iters = torch.empty(R, device=X.device, dtype=torch.int32)
    labels = torch.empty(W, device=X.device, dtype=torch.int32)
    with torch.cuda.device(X.device):
        L.check(L.load().dsk_vbx(X.data_ptr(), W, d, off.data_ptr(), R, lab.data_ptr(), S, phi.data_ptr(), float(Fa),
                                 float(Fb), float(loop_p), float(init_smoothing), int(max_iters), float(epsilon),
                                 gamma.data_ptr(), pi.data_ptr(), elbo.data_ptr(), iters.data_ptr(), labels.data_ptr(),
                                 L.cur_stream()), "dsk_vbx")
    return gamma, pi, elbo, iters, labels
