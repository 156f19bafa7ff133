"""Oracles of the batch-hard triplet loss — TEST INFRASTRUCTURE ONLY (the product never imports this module).

* ``batch_hard_triplet``: ctypes wrapper of oracle/batch_hard_oracle.c, the step-by-step fp32 restatement of the
  selection, its tie rules and the fixed-order mean (bit-exact target of dsk_batch_hard_triplet).
* ``batch_hard_loss``: fp64-capable torch-autograd restatement of the loss with the selection GIVEN, for gradient
  checks (the selection is piecewise constant in E, so the gradient is taken with the engine's choice pinned).

The reference has no batch-hard loss: parity with it is unpinned.
"""
import ctypes
import os
import subprocess

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "batch_hard_oracle.c")
OUT_DIR = os.path.join(_HERE, "_build")
LIB = os.path.join(OUT_DIR, "libbatch_hard_oracle.so")
_lib = None


def build(force=False):
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= os.path.getmtime(SRC):
        return LIB
    os.makedirs(OUT_DIR, exist_ok=True)
    cmd = ["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", LIB, SRC, "-lm"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError("gcc failed: " + r.stderr)
    return LIB


def load():
    global _lib
    if _lib is None:
        try:
            build()
        except Exception:
            if not os.path.exists(LIB):
                raise
        _lib = ctypes.CDLL(LIB)
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def batch_hard_triplet(E, labels, margin):
    """-> (loss float32, pos_idx int64, neg_idx int64, d_ap float32, d_an float32, valid bool), numpy."""
    E = np.ascontiguousarray(E, dtype=np.float32)
    labels = np.ascontiguousarray(labels, dtype=np.int64)
    N, D = E.shape
    loss = np.empty(1, np.float32)
    pos, neg = np.empty(N, np.int64), np.empty(N, np.int64)
    d_ap, d_an = np.empty(N, np.float32), np.empty(N, np.float32)
    valid = np.empty(N, np.uint8)
    load().orc_batch_hard_triplet(_p(E), _p(labels), N, D, ctypes.c_float(margin), _p(loss), _p(pos), _p(neg),
                                  _p(d_ap), _p(d_an), _p(valid))
    return loss[0], pos, neg, d_ap, d_an, valid.astype(bool)


def batch_hard_loss(E, pos_idx, neg_idx, valid, margin):
    """Differentiable loss with the selection given: (1/V) sum_{valid i} clamp(margin + d(i,p_i) - d(i,n_i), 0),
    d = PairwiseDistance (reference model.py:13-18, eps 1e-4/D); 0 when V = 0.  Runs in E's dtype (use fp64)."""
    N, D = E.shape
    valid = torch.as_tensor(valid, dtype=torch.bool)
    ar = torch.arange(N)
    p = torch.where(valid, torch.as_tensor(pos_idx), ar)     # invalid anchors: any in-range index, masked out below
    n = torch.where(valid, torch.as_tensor(neg_idx), ar)
    eps = 1e-4 / D
    d_ap = torch.sqrt(((E - E[p]) ** 2).sum(1) + eps)
    d_an = torch.sqrt(((E - E[n]) ** 2).sum(1) + eps)
    h = torch.clamp(margin + d_ap - d_an, min=0.0) * valid.to(E.dtype)
    V = int(valid.sum())
    return h.sum() / max(V, 1)
