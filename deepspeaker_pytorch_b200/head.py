"""Classifier head and cross-entropy of the reference's hard-triplet branch on repo kernels (no cuBLAS / ATen math).

* ``LinearFn``          — ``model.classifier`` = ``nn.Linear(embedding_size, num_classes)`` applied by
  ``DeepSpeakerModel.forward_classifier`` (reference model.py:167,220-223)
* ``CrossEntropyLoss``  — ``nn.CrossEntropyLoss()`` as the reference's train loop uses it
  (reference train_triplet.py:281-285): mean over rows of ``logsumexp(logits) - logits[label]``

Both are ``torch.autograd.Function``s over the C ABI (``dsk_linear_*``, ``dsk_cross_entropy*``): fp32, fixed
summation order (deterministic), asynchronous on the current stream, loss returned as a device scalar.
"""
from __future__ import annotations

import torch

from . import _lib as L


def _cuda_f32(t, what):
    if not t.is_cuda:
        raise RuntimeError(f"{what}: CUDA tensors required; there is no CPU fallback")
    return t.detach().float().contiguous()


class LinearFn(torch.autograd.Function):
    """y = x @ w.T + b — model.py:167 applied at :222."""

    @staticmethod
    def forward(ctx, x, w, b):
        xc, wc = _cuda_f32(x, "linear"), _cuda_f32(w, "linear")
        bc = None if b is None else _cuda_f32(b, "linear")
        M, K = xc.shape
        N = wc.shape[0]
        if wc.shape[1] != K:
            raise RuntimeError(f"linear: x is (M,{K}) but weight is {tuple(wc.shape)}")
        y = torch.empty(M, N, device=x.device, dtype=torch.float32)
        if M > 0:
            with torch.cuda.device(x.device):
                L.check(L.load().dsk_linear_forward(xc.data_ptr(), wc.data_ptr(), L.ptr(bc), M, N, K, y.data_ptr(),
                                                    L.cur_stream()), "dsk_linear_forward")
        ctx.save_for_backward(xc, wc)
        ctx.has_bias = b is not None
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w = ctx.saved_tensors
        M, K = x.shape
        N = w.shape[0]
        gy = _cuda_f32(gy, "linear backward")
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        gw = torch.empty_like(w) if ctx.needs_input_grad[1] else None
        gb = torch.empty(N, device=x.device, dtype=torch.float32) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        if M == 0:
            for t in (gx, gw, gb):
                if t is not None:
                    t.zero_()
            return gx, gw, gb
        with torch.cuda.device(x.device):
            L.check(L.load().dsk_linear_backward(x.data_ptr(), w.data_ptr(), gy.data_ptr(), M, N, K, L.ptr(gx), L.ptr(gw),
                                                 L.ptr(gb), L.cur_stream()), "dsk_linear_backward")
        return gx, gw, gb


class CrossEntropyFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels):
        lg = _cuda_f32(logits, "cross_entropy")
        if lg.dim() != 2:
            raise RuntimeError("cross_entropy: expected (M, C) logits")
        M, C = lg.shape
        if M == 0:
            raise RuntimeError("cross_entropy: empty batch")
        lab = labels.to(device=lg.device, dtype=torch.int64).contiguous()
        if lab.shape != (M,):
            raise RuntimeError(f"cross_entropy: labels must be ({M},), got {tuple(lab.shape)}")
        loss = torch.empty(1, device=lg.device, dtype=torch.float32)
        lse = torch.empty(M, device=lg.device, dtype=torch.float32)
        rows = torch.empty(M, device=lg.device, dtype=torch.float32)
        with torch.cuda.device(lg.device):
            L.check(L.load().dsk_cross_entropy(lg.data_ptr(), lab.data_ptr(), M, C, loss.data_ptr(), lse.data_ptr(),
                                               rows.data_ptr(), L.cur_stream()), "dsk_cross_entropy")
        ctx.save_for_backward(lg, lab, lse)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, gl):
        lg, lab, lse = ctx.saved_tensors
        M, C = lg.shape
        gl = gl.detach().float().reshape(1).contiguous()
        d = torch.empty_like(lg)
        with torch.cuda.device(lg.device):
            L.check(L.load().dsk_cross_entropy_bwd(lg.data_ptr(), lab.data_ptr(), lse.data_ptr(), gl.data_ptr(), M, C,
                                                   d.data_ptr(), L.cur_stream()), "dsk_cross_entropy_bwd")
        return d, None


class CrossEntropyLoss:
    """Drop-in for the ``nn.CrossEntropyLoss()`` instance of train_triplet.py:281 (default arguments: mean reduction,
    no class weights, no label smoothing) — callable and with ``.forward`` like the module it replaces."""

    def forward(self, input, target):
        return CrossEntropyFn.apply(input, target)

    __call__ = forward

    def cuda(self, *a, **k):   # nn.Module-style chaining used by some forks of the reference
        return self
