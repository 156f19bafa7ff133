"""Train-mode forward/backward of DeepSpeakerModel on the H100 engine.

Mirrors what autograd does for the reference when the module is in train mode
(reference train_triplet.py:203,215-224): BatchNorm uses the batch statistics of each call, running
statistics are updated in place, and ``loss.backward()`` produces gradients for the 12 conv weights, the 12
BatchNorm affine pairs and fc (the classifier is outside this path and gets no gradient, SURVEY §0 fact 5).
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib as L
from .engine import conv_bn_modules


def _train_params(module):
    """The 38 parameters the path differentiates, in a fixed order: 12 x (conv.weight, bn.weight, bn.bias), fc.weight, fc.bias."""
    ps = []
    for conv, bn in conv_bn_modules(module):
        ps += [conv.weight, bn.weight, bn.bias]
    ps += [module.model.fc.weight, module.model.fc.bias]
    return ps


class _CtxGuard:
    """Returns the library-side context to the pool if the autograd graph is dropped without a backward."""

    def __init__(self, engine, tctx):
        self.engine, self.tctx, self.live = engine, tctx, True

    def consume(self):
        self.live = False

    def __del__(self):
        try:
            if self.live and self.engine.handle.value:
                self.engine.lib.dsk_train_ctx_release(self.engine.handle, self.tctx)
        except Exception:
            pass


class TrainForwardFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, engine, *params):
        B, _, T, _ = x.shape
        emb = torch.empty(B, engine.module_ref.embedding_size, device=x.device, dtype=torch.float32)
        tctx = ctypes.c_void_p()
        L.check(engine.lib.dsk_rescnn_forward_train(engine.handle, x.data_ptr(), B, T, emb.data_ptr(), ctypes.byref(tctx),
                                                    L.cur_stream()), "dsk_rescnn_forward_train")
        ctx.engine = engine
        ctx.guard = _CtxGuard(engine, tctx)
        ctx.save_for_backward(x, *params)  # x must outlive the backward (conv1's weight gradient reads it)
        return emb

    @staticmethod
    def backward(ctx, grad_emb):
        engine = ctx.engine
        saved = ctx.saved_tensors
        params = saved[1:]
        grads = engine.grad_scratch(params)
        g = _grads_struct(grads)
        ge = grad_emb.float().contiguous()
        with torch.cuda.device(ge.device):
            L.check(engine.lib.dsk_rescnn_backward(engine.handle, ctx.guard.tctx, ge.data_ptr(), ctypes.byref(g),
                                                   L.cur_stream()), "dsk_rescnn_backward")
        ctx.guard.consume()
        return (None, None) + tuple(grads)


def _forward_one(engine, x, params, need_grad):
    """One train-mode forward on the CURRENT stream.  Returns (emb, library context or None if already released)."""
    if need_grad:
        emb = TrainForwardFn.apply(x, engine, *params)
        return emb, emb.grad_fn.guard.tctx
    B, _, T, _ = x.shape
    emb = torch.empty(B, engine.module_ref.embedding_size, device=x.device, dtype=torch.float32)
    tctx = ctypes.c_void_p()
    L.check(engine.lib.dsk_rescnn_forward_train(engine.handle, x.data_ptr(), B, T, emb.data_ptr(), ctypes.byref(tctx),
                                                L.cur_stream()), "dsk_rescnn_forward_train")
    return emb, tctx


def _grads_struct(views):
    """The ``dsk_grads`` output pointers of a backward: the 38 gradient tensors in ``_train_params`` order."""
    g = L.DskGrads()
    for i in range(L.DSK_NUM_CONV):
        g.conv_w[i] = views[3 * i].data_ptr()
        g.bn_gamma[i] = views[3 * i + 1].data_ptr()
        g.bn_beta[i] = views[3 * i + 2].data_ptr()
    g.fc_w = views[-2].data_ptr()
    g.fc_b = views[-1].data_ptr()
    return g


def forward_train(engine, x):
    module = engine.module_ref
    if sync_bn_setting(module)[0]:
        return forward_train_many(engine, [x])[0]
    engine.sync_weights(eval_mode=False)
    engine.train_calls += 1  # running statistics are about to change: invalidates the eval-mode BN fold
    params = _train_params(module)
    need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in params)
    emb, tctx = _forward_one(engine, x, params, need_grad)
    if not need_grad:
        L.check(engine.lib.dsk_train_ctx_release(engine.handle, tctx), "dsk_train_ctx_release")
    # nn.BatchNorm2d bookkeeping in train mode
    torch._foreach_add_([bn.num_batches_tracked for _, bn in conv_bn_modules(module)], 1)
    return emb


class TripletForwardFn(torch.autograd.Function):
    """The K train-mode forwards of one step as ONE autograd node.  Forward: call k on side stream k.  Backward: the K
    backward chains on the same K streams, each into its own flat gradient buffer, then ONE ordered sum of the flat
    buffers on the caller's stream.  K separate nodes gave the same numbers, but autograd then summed the three
    gradients of each of the 38 parameters itself: 114 small ``add`` launches at the end of every step, serial, after the
    last backward kernel.  The sum here runs in the order autograd used (last
    call first: (g_n + g_p) + g_a), so the gradients are the same bits as those of K sequential calls."""

    @staticmethod
    def forward(ctx, engine, k, *args):
        xs, params = args[:k], args[k:]
        outs, tctxs = _launch_many(engine, xs)
        ctx.engine, ctx.k, ctx.params = engine, k, params
        ctx.guards = [_CtxGuard(engine, t) for t in tctxs]
        ctx.out_shape = outs[0].shape
        ctx.save_for_backward(*xs, *params)  # the inputs must outlive the backward (conv1's weight gradient reads them)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grad_embs):
        engine, k, params = ctx.engine, ctx.k, ctx.params
        _ = ctx.saved_tensors                      # raises if a parameter was modified in place since the forward
        dev = engine.device
        with torch.cuda.device(dev):
            cur = torch.cuda.current_stream(dev)
            flats, views = [], None
            for ge, st, guard in zip(grad_embs, engine.side_streams, ctx.guards):
                ge = (torch.zeros(ctx.out_shape, device=dev, dtype=torch.float32) if ge is None
                      else ge.float().contiguous())
                flat, views = engine.grad_scratch(params, with_flat=True)
                g = _grads_struct(views)
                st.wait_stream(cur)                # grad_emb was produced on the caller's stream
                with torch.cuda.stream(st):
                    L.check(engine.lib.dsk_rescnn_backward(engine.handle, guard.tctx, ge.data_ptr(), ctypes.byref(g),
                                                           L.cur_stream()), "dsk_rescnn_backward")
                guard.consume()
                flats.append(flat)
            for st in engine.side_streams[:k]:
                cur.wait_stream(st)                # also keeps every grad_emb alive long enough: it is freed on `cur`
            return _sum_grads(ctx, engine, params, flats, views, 2 + k)


def _sum_grads(node, engine, params, flats, views, n_inputs):
    """The end of a K-call backward: ONE ordered sum of the K flat gradient buffers into the last one, whose ``views``
    these are, in autograd's order for K separate calls (last call first: (g_n + g_p) + g_a).  Returns ``node``'s
    backward result for its ``n_inputs`` non-parameter inputs followed by the parameters."""
    acc = flats[-1]
    for f in reversed(flats[:-1]):
        acc.add_(f)
    # parameters whose .grad is a view of an optimizer / data-parallel bucket (FusedAdagrad, GradBucket):
    # accumulate into the bucket with one multi-tensor add instead of 38 AccumulateGrad nodes
    if (all(p.grad is not None and p.grad is getattr(p, "_dsk_bucket_grad", None) for p in params)
            and _engine_accumulates_into(node, params)):
        torch._foreach_add_([p.grad for p in params], list(views))
        engine.bucket_accumulations += 1
        return (None,) * (n_inputs + len(params))
    return (None,) * n_inputs + tuple(views)


def _engine_accumulates_into(node, params):
    """True when the running backward will accumulate this node's parameter gradients into ``p.grad`` (``loss.backward()``),
    False when it captures them instead (``torch.autograd.grad``: the AccumulateGrad nodes are not executed and the query
    raises) - then the gradients must be returned to autograd, not added into the bucket."""
    try:
        acc = {id(fn.variable): fn for fn, _ in node.next_functions if fn is not None and hasattr(fn, "variable")}
        return all(id(p) in acc and torch._C._will_engine_execute_node(acc[id(p)]) for p in params)
    except Exception:
        return False


def _launch_many(engine, xs):
    """Forward k of ``xs`` on side stream k, running-statistics updates deferred; joins the side streams.  Returns
    (embeddings, library contexts)."""
    dev = engine.device
    cur = torch.cuda.current_stream(dev)
    while len(engine.side_streams) < len(xs):
        engine.side_streams.append(torch.cuda.Stream(dev))
    L.check(engine.lib.dsk_set_defer_running_stats(engine.handle, 1), "dsk_set_defer_running_stats")
    outs, ctxs = [], []
    try:
        for x, st in zip(xs, engine.side_streams):
            st.wait_stream(cur)                      # inputs (and the parameters) were produced on the caller's stream
            with torch.cuda.stream(st):
                emb, tctx = _forward_one(engine, x, None, False)
            x.record_stream(st)
            outs.append(emb)
            ctxs.append(tctx)
    finally:
        L.check(engine.lib.dsk_set_defer_running_stats(engine.handle, 0), "dsk_set_defer_running_stats")
    for st, emb in zip(engine.side_streams, outs):
        cur.wait_stream(st)
        emb.record_stream(cur)
    return outs, ctxs


def forward_train_many(engine, xs):
    """Several independent train-mode forwards of one step (the anchor / positive / negative calls of
    train_triplet.py:215) as ONE autograd node.  By default the calls are IN FLIGHT TOGETHER: forward k runs on its own
    side stream, so the HBM-bound BatchNorm passes of one call overlap the tensor-core convs of another, and so do the
    three backwards (``TripletForwardFn``).  With synchronised BatchNorm they run in lockstep on the current stream
    (``SyncTrainForwardFn``): one collective per stage carries every call's records, and every rank must call this with
    the same number of forwards of the same batch size (a group of None is this process alone, on the same staged path,
    so results never depend on the number of ranks).  Results are those of the sequential calls, bit for bit: batch
    statistics are per call anyway, the running-statistics updates are committed in call order
    (``dsk_train_ctx_commit_stats``), and the gradients are summed in autograd's order."""
    module = engine.module_ref
    on, group = sync_bn_setting(module)
    node, launch, args = (SyncTrainForwardFn, _sync_forward, (group,)) if on else (TripletForwardFn, _launch_many, ())
    engine.sync_weights(eval_mode=False)
    engine.train_calls += 1
    params = _train_params(module)
    need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in params)
    xs = [x.contiguous().float() for x in xs]
    if need_grad:
        outs = list(node.apply(engine, *args, len(xs), *xs, *params))
        ctxs = [g.tctx for g in outs[0].grad_fn.guards]
    else:
        outs, ctxs = launch(engine, xs, *args)
    for tctx in ctxs:                                # momentum updates in call order, on the caller's stream
        L.check(engine.lib.dsk_train_ctx_commit_stats(engine.handle, tctx, L.cur_stream()), "dsk_train_ctx_commit_stats")
        if not need_grad:
            L.check(engine.lib.dsk_train_ctx_release(engine.handle, tctx), "dsk_train_ctx_release")
    torch._foreach_add_([bn.num_batches_tracked for _, bn in conv_bn_modules(module)], len(xs))
    return outs


# ---- synchronised BatchNorm ------------------------------------------------------------------------------------------
# DeepSpeakerModel.sync_batchnorm(group): every train-mode BatchNorm layer normalises with the statistics of the GLOBAL
# batch of all ranks.  The library runs the forward and the backward as resumable stages (include/dsk.h, dsk_sync_*);
# at each of the 12 forward and 13 backward exchange points a stage generator below yields this rank's per-utterance
# records (a uint8 device tensor) and receives the records of every rank's utterances, concatenated in rank order.
# ``run_lockstep`` drives several generators through one exchange per stage; ``parallel.gather_records`` is the exchange
# of a process group (one all_gather_into_tensor).

def sync_bn_setting(module):
    """(on, process group) of ``DeepSpeakerModel.sync_batchnorm``."""
    s = getattr(module, "_sync_bn", None)
    return (False, None) if s is None else (True, s[0])


class _DeviceBytes:
    """A library-owned device buffer as a zero-copy uint8 tensor (``torch.as_tensor`` reads this interface)."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "strides": None,
                                         "version": 2}


def _stage_loop(engine, tctx, B):
    more = ctypes.c_int32(1)
    while more.value:
        p, nb = ctypes.c_void_p(), ctypes.c_int64()
        L.check(engine.lib.dsk_sync_records(engine.handle, tctx, ctypes.byref(p), ctypes.byref(nb)), "dsk_sync_records")
        local = torch.as_tensor(_DeviceBytes(p.value, nb.value), device=engine.device)
        gathered = yield local
        if gathered.dtype != torch.uint8 or gathered.numel() % (nb.value // B):
            raise ValueError("gathered records must be the uint8 records of whole utterances")
        n_total = gathered.numel() // (nb.value // B)
        L.check(engine.lib.dsk_sync_stage(engine.handle, tctx, gathered.data_ptr(), n_total, ctypes.byref(more),
                                          L.cur_stream()), "dsk_sync_stage")


def sync_forward_stages(engine, x, emb):
    """Generator of one synchronised train-mode forward of ``x`` (B, 1, T, 64) into ``emb`` (B, E) on the current
    stream: yields this rank's records 12 times, each time receiving the gathered records (uint8, rank order); returns
    the library context (StopIteration.value), which the backward stages consume."""
    B, _, T, _ = x.shape
    tctx = ctypes.c_void_p()
    L.check(engine.lib.dsk_sync_forward_begin(engine.handle, x.data_ptr(), B, T, emb.data_ptr(), ctypes.byref(tctx),
                                              L.cur_stream()), "dsk_sync_forward_begin")
    done = False
    try:
        yield from _stage_loop(engine, tctx, B)
        done = True
    finally:
        if not done:
            engine.lib.dsk_train_ctx_release(engine.handle, tctx)
    return tctx


def sync_backward_stages(engine, tctx, B, grad_emb, views):
    """Generator of the backward of a synchronised forward: 13 exchanges (the loss scale, then BatchNorm layers 11..0).
    The 38 parameter gradients are written into ``views``: dgamma / dbeta and the weight gradients are this rank's
    share, which the data-parallel gradient reduction adds up."""
    g = _grads_struct(views)
    L.check(engine.lib.dsk_sync_backward_begin(engine.handle, tctx, grad_emb.data_ptr(), ctypes.byref(g), L.cur_stream()),
            "dsk_sync_backward_begin")
    yield from _stage_loop(engine, tctx, B)


def run_lockstep(gens, exchange):
    """Drives stage generators that exchange at the same points: ``exchange(list of local records)`` returns one
    gathered record tensor per generator.  One exchange per stage for all of them.  Returns the generators' results."""
    local = [next(g) for g in gens]
    while True:
        gathered = exchange(local)
        nxt, results = [], []
        for g, rec in zip(gens, gathered):
            try:
                nxt.append(g.send(rec))
            except StopIteration as stop:
                results.append(stop.value)
        if len(results) == len(gens):
            return results
        if results:
            raise RuntimeError("synchronised stage generators fell out of step")
        local = nxt


def _sync_forward(engine, xs, group):
    """The synchronised forwards of ``xs`` in lockstep on the current stream: one exchange per stage for all of them.
    With several forwards the running-statistics updates are deferred (committed afterwards in call order)."""
    from .parallel import gather_records

    embs = [torch.empty(x.shape[0], engine.module_ref.embedding_size, device=x.device, dtype=torch.float32) for x in xs]
    gens = [sync_forward_stages(engine, x, e) for x, e in zip(xs, embs)]
    defer = len(xs) > 1
    if defer:
        L.check(engine.lib.dsk_set_defer_running_stats(engine.handle, 1), "dsk_set_defer_running_stats")
    try:
        ctxs = run_lockstep(gens, lambda local: gather_records(local, group))
    finally:
        if defer:
            L.check(engine.lib.dsk_set_defer_running_stats(engine.handle, 0), "dsk_set_defer_running_stats")
    return embs, ctxs


class SyncTrainForwardFn(torch.autograd.Function):
    """K synchronised train-mode forwards of one step (K = 1 for ``model(x)``, 3 for ``forward_triplet``) as ONE
    autograd node.  Forward and backward drive the K stage generators in lockstep, so a stage's K record sets travel in
    one collective; the backward's collectives therefore run inside ``loss.backward()``, and every rank must run the
    same backward.  The K gradients are summed as ``TripletForwardFn`` sums them (last call first), into an optimizer /
    data-parallel bucket directly when the parameters' gradients are views of one."""

    @staticmethod
    def forward(ctx, engine, group, k, *args):
        xs, params = args[:k], args[k:]
        outs, tctxs = _sync_forward(engine, xs, group)
        ctx.engine, ctx.group, ctx.k, ctx.params = engine, group, k, params
        ctx.guards = [_CtxGuard(engine, t) for t in tctxs]
        ctx.out_shapes = [o.shape for o in outs]
        ctx.save_for_backward(*xs, *params)  # the inputs must outlive the backward (conv1's weight gradient reads them)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grad_embs):
        from .parallel import gather_records

        engine, k, params = ctx.engine, ctx.k, ctx.params
        _ = ctx.saved_tensors
        dev = engine.device
        with torch.cuda.device(dev):
            flats, views, ges, gens = [], None, [], []
            for ge, shape, guard in zip(grad_embs, ctx.out_shapes, ctx.guards):
                ge = torch.zeros(shape, device=dev, dtype=torch.float32) if ge is None else ge.float().contiguous()
                flat, views = engine.grad_scratch(params, with_flat=True)
                gens.append(sync_backward_stages(engine, guard.tctx, shape[0], ge, views))
                ges.append(ge)
                flats.append(flat)
            run_lockstep(gens, lambda local: gather_records(local, ctx.group))
            for guard in ctx.guards:
                guard.consume()
            return _sum_grads(ctx, engine, params, flats, views, 3 + k)
