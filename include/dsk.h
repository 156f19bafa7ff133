/*
 * dsk.h — C ABI of the H100-native Deep Speaker hot path (libdsk.so).
 *
 * The reference (qqueing/DeepSpeaker-pytorch) is 100 % Python and reaches the GPU only through
 * torch.nn library calls; it has no FFI of its own.  Each entry point below therefore cites the
 * reference *Python* call site whose arithmetic it replaces (file:line in the reference project).
 * A maintainer binds these with ctypes (see INTEGRATION.md); the host-side mirror of the
 * reference's classes lives in deepspeaker_pytorch_b200/model.py.
 *
 * Conventions
 *  - every pointer is a raw CUDA device pointer owned by the caller (PyTorch); the library
 *    borrows it for the duration of the call and never frees it;
 *  - every function is asynchronous on `stream` (a cudaStream_t passed as void*), never
 *    synchronises the device and never reads results on the host;
 *  - return value: 0 on success, negative dsk_status on error; dsk_last_error() gives the
 *    message of the last failure on the calling thread;
 *  - no exceptions cross this boundary, there is no CPU fallback.
 */
#ifndef DSK_H_
#define DSK_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  DSK_OK = 0,
  DSK_ERR_INVALID = -1, /* bad argument / unsupported shape */
  DSK_ERR_CUDA = -2,    /* a CUDA runtime / driver call failed */
  DSK_ERR_STATE = -3,   /* call sequence error (e.g. forward before load_weights) */
  DSK_ERR_ARCH = -4     /* device is not sm_90 */
} dsk_status;

/* 16-bit tensor-core operand format (fp32 accumulation either way) */
typedef enum { DSK_F16 = 0, DSK_BF16 = 1 } dsk_operand_t;

/* BatchNorm behaviour of a forward: running statistics (eval) or batch statistics (train) */
typedef enum { DSK_EVAL = 0, DSK_TRAIN = 1 } dsk_mode_t;

#define DSK_NUM_CONV 12 /* conv1, layer1.0.conv1, layer1.0.conv2, conv2, layer2.0.conv1, ... layer4.0.conv2 */

/* Parameters of DeepSpeakerModel.model (fp32, PyTorch layouts), reference model.py:91-112,162-164.
 * conv_w[i]: OIHW.  i = 3*stage + {0: convK (5x5 s2), 1: layerK.0.conv1, 2: layerK.0.conv2 (3x3)}.
 * bn_*[i]  : the BatchNorm2d that follows conv i (bnK, layerK.0.bn1, layerK.0.bn2).
 * fc_w     : (embedding_size, 2048) with column index c*4 + w (model.py:164,208-209). */
typedef struct {
  const float* conv_w[DSK_NUM_CONV];
  const float* bn_gamma[DSK_NUM_CONV];
  const float* bn_beta[DSK_NUM_CONV];
  float* bn_running_mean[DSK_NUM_CONV]; /* read in eval; updated in place in train (momentum 0.1) */
  float* bn_running_var[DSK_NUM_CONV];
  const float* fc_w;
  const float* fc_b;
  int32_t embedding_size; /* 512 */
} dsk_weights;

/* Gradients, same layouts as dsk_weights (fp32, written not accumulated). */
typedef struct {
  float* conv_w[DSK_NUM_CONV];
  float* bn_gamma[DSK_NUM_CONV];
  float* bn_beta[DSK_NUM_CONV];
  float* fc_w;
  float* fc_b;
} dsk_grads;

typedef struct dsk_handle_s* dsk_handle;
typedef struct dsk_train_ctx_s* dsk_train_ctx; /* what one train-mode forward saved for its backward */
typedef struct dsk_pipeline_s* dsk_pipeline;   /* serving pipeline: copy streams + compute lanes around one weight image */

const char* dsk_last_error(void);
int32_t dsk_version(void);

/* Per-module engine state (repacked weights, folded BN, workspace, TMA descriptors).
 * Created at DeepSpeakerModel.cuda()/first call, released in __del__ (model.py:153-167). */
int32_t dsk_create(dsk_handle* out, int32_t device, int32_t operand /* dsk_operand_t */);
int32_t dsk_destroy(dsk_handle h);

/* Repack conv weights to [tap][cout][cin] 16-bit, fold eval BatchNorm to scale/bias, reorder fc.
 * Must be called after every parameter update (the Python shim tracks parameter versions). */
int32_t dsk_load_weights(dsk_handle h, const dsk_weights* w, void* stream);
/* The same for a handle that is about to TRAIN (every optimizer step changes every parameter, so this runs once per
 * step, before the forwards): rebuilds only what dsk_rescnn_forward_train / dsk_rescnn_backward read - the forward and
 * data-gradient operand images of the eleven tensor-core convs (one kernel launch), conv1's filter and the reordered fc
 * weight - and skips the eval-only work (BatchNorm folding, conv1's split image, the plane-major 5x5 images).
 * dsk_rescnn_forward (eval) then fails with DSK_ERR_STATE until dsk_load_weights is called again. */
int32_t dsk_load_weights_train(dsk_handle h, const dsk_weights* w, void* stream);
/* Serving with several forwards in flight (one handle + activation workspace per compute stream): `h` borrows the
 * packed weights / folded BN of `src` instead of holding its own copy, so all lanes read one 21 MB weight image (it
 * has to stay L2-resident: the convs re-read it per tile).  `h` follows later dsk_load_weights(src) calls at its next
 * forward; it is inference-only, must not be given weights of its own, and `src` must outlive it. */
int32_t dsk_share_weights(dsk_handle h, dsk_handle src);

/* DeepSpeakerModel.forward (reference model.py:185-218), BN in eval mode
 * (train_triplet.py:332,347): x (B,1,T,64) fp32 contiguous -> emb (B,E) fp32 with ||emb||=10.
 * T must be a multiple of 16.
 * An utterance's embedding, and every activation of it, has the same bits whatever else is in the batch (its size,
 * order and content) under the default whole-tile scheduling; DSK_STREAM_K=1 cuts each tile's K loop where the tile
 * count puts it, which can move the last bits.  Nothing else bounds B and T: the workspace grows with B * T (130 MiB at
 * 64 x 160), and the halo convs' 32-bit position arithmetic is exact for every shape whose workspace fits in 80 GiB (a
 * layer past 2^31 padded positions fails with DSK_ERR_INVALID).
 * Non-finite input: a NaN or +-inf element of x makes that utterance's embedding all NaN (every activation is NaN
 * exactly where a conv window reaches it, in every channel; the clamps keep NaN, as Hardtanh does) and leaves every
 * other utterance's bits unchanged; pads stay +0.  conv1 splits x into 16-bit halves x_hi + x_lo, so the finite input
 * range is per operand type: fp16 |x| < 65520 (past it x_hi is inf and the element acts as a NaN), bf16 every finite
 * fp32.  An infinite element gives NaN too, where the reference's fp32 conv would carry +-inf into its clamp.  A NaN
 * running statistic makes every embedding NaN, as nn.BatchNorm2d in eval does.
 * Asynchronous on `stream`, with one exception that synchronises the DEVICE: the first forward after
 * dsk_load_weights (the folded BN affine is copied to the host and baked into the conv kernels' parameter block).
 * The first call of a new (B, T) shape rebuilds the plan and re-zeroes the padded activation workspace with a
 * memset ORDERED ON `stream` (after the forwards this handle still has in flight there); if the workspace has to
 * grow, cudaFree synchronises the device.  One handle must only be driven from one stream at a time (use one handle
 * per compute lane, dsk_share_weights).  From the second call of a shape on, the 15 kernels are replayed as one CUDA graph whose first / last
 * nodes are re-pointed at x / emb; inside a caller's own stream capture the plain launches are recorded instead (warm the
 * shape up before capturing). */
int32_t dsk_rescnn_forward(dsk_handle h, const float* x, int32_t B, int32_t T, float* emb, int32_t mode,
                           void* stream);

/* DeepSpeakerModel.forward with the module in train mode (train_triplet.py:203,215): BatchNorm uses the batch
 * statistics of THIS call (the reference forwards a, p and n separately, so statistics are per call) and updates
 * running_mean / running_var in place (momentum 0.1, unbiased variance).  Saves activations in *ctx for
 * dsk_rescnn_backward; x must stay alive until then.  Contexts are pooled inside the handle.
 * A non-finite element of any utterance makes the batch statistics NaN, so every embedding of the call and the running
 * statistics become NaN, as in torch; nothing is clamped back to a number. */
int32_t dsk_rescnn_forward_train(dsk_handle h, const float* x, int32_t B, int32_t T, float* emb, dsk_train_ctx* ctx,
                                 void* stream);
/* Several train-mode forwards of one step in flight at once (DeepSpeakerModel.forward_triplet runs the anchor / positive /
 * negative forwards of train_triplet.py:215 on three streams so that the HBM-bound BatchNorm passes of one overlap the
 * tensor-core convs of another): with `on` != 0 a train forward only RECORDS its batch statistics in the context and
 * leaves running_mean / running_var alone; dsk_train_ctx_commit_stats then applies that forward's momentum update
 * (all 12 layers, one launch).  Committing the contexts in the order of the reference's sequential calls (a, p, n) on
 * one stream gives bit-identical running statistics.  A context must be committed before its backward consumes it. */
int32_t dsk_set_defer_running_stats(dsk_handle h, int32_t on);
int32_t dsk_train_ctx_commit_stats(dsk_handle h, dsk_train_ctx ctx, void* stream);
/* Backward of that forward (what loss.backward() triggers, train_triplet.py:223): grad_emb (B,E) fp32 ->
 * gradients of every conv / BN / fc parameter, written (not accumulated) into `grads`.  Consumes the context. */
int32_t dsk_rescnn_backward(dsk_handle h, dsk_train_ctx ctx, const float* grad_emb, const dsk_grads* grads,
                            void* stream);
/* Debug / test read-back of what a train-mode forward saved: which = 0 the pre-BatchNorm conv output (fp32),
 * 1 the post-activation tensor (16-bit), of conv layer `layer` (0..11), converted to fp32 NCHW. */
int32_t dsk_train_ctx_read(dsk_handle h, dsk_train_ctx ctx, int32_t which, int32_t layer, float* out_nchw, void* stream);
/* Debug / test: the plan the backward of `ctx` (as bound by its last forward) uses for conv layer `layer` (0..11):
 * out[0] = K splits of the weight-gradient GEMM, out[1] = 128-pixel chunks per split (both 0 for conv1),
 * out[2] = partial-sum blocks per 64-channel group of the BatchNorm reductions (forward statistics and backward sums of
 * the unsynchronised path).  Host-only: no device work. */
int32_t dsk_debug_backward_plan(dsk_handle h, dsk_train_ctx ctx, int32_t layer, int32_t* out);
/* Debug / test read-back: activation `layer` (0..11: output of conv `layer` after BN, residual and clip) of this handle's
 * most recent dsk_rescnn_forward, byte for byte as stored: 16-bit zero-padded NHWC (dsk_padded_positions(B,H,W) * C),
 * or parity-planar (4 planes of dsk_padded_positions(B,H/2,W/2) * C) for the block outputs that feed a stride-2 conv.
 * *planar_out says which; dst_bytes must equal that size.  Ordered on `stream`.  DSK_ERR_STATE if no plan is cached. */
int32_t dsk_debug_read_eval_activation(dsk_handle h, int32_t layer, void* dst, int64_t dst_bytes, int32_t* planar_out,
                                       void* stream);
/* Return an unused context to the pool (forward without backward, e.g. under no_grad). */
int32_t dsk_train_ctx_release(dsk_handle h, dsk_train_ctx ctx);
/* fp16 operands: inside the backward the 16-bit gradient tensors are multiplied by a power of two S and every parameter
 * gradient is divided by it again.  scale = 0 (default): S is chosen PER BACKWARD ON THE DEVICE from the largest incoming
 * gradient, S = 2^floor(log2(512 / max|dL/d(fc output)|)) - no host synchronisation, follows the loss as it shrinks during
 * training; scale > 0: that fixed value.  bf16 operands: 1 unless set. */
int32_t dsk_set_loss_scale(dsk_handle h, float scale);

/* Synchronised BatchNorm under data parallelism: the train forward and backward as resumable stages, so that the caller
 * can exchange per-utterance records between ranks at every BatchNorm layer (the library issues no collective).  Every
 * layer normalises with the statistics of the GLOBAL batch, combined in global utterance order: what a rank computes for
 * its own utterances is bit-identical for every way of splitting the batch over ranks, one rank included.
 *
 *   dsk_sync_forward_begin   conv1 and layer 0's records; *ctx is a pooled train context
 *   dsk_sync_backward_begin  (after the forward's last stage) the l2-norm backward and the loss-scale records
 *   dsk_sync_records         device pointer and byte size of this stage's records of the B local utterances
 *   dsk_sync_stage           consumes the records of all n_total utterances, gathered in rank order, and runs up to the
 *                            next exchange; *more = 0 after the forward's tail (emb written) / layer 0's weight gradient
 *
 * The forward has 12 exchanges (one per BatchNorm layer), the backward 13 (the loss scale, then layers 11..0).  Records,
 * fp32 words per utterance (u in rank order, C the layer's channels):
 *   forward, layer i:  3C + 1: [0,C) pivot k_c = the utterance's first pixel of channel c, [C,2C) sum (x - k_c),
 *                      [2C,3C) sum (x - k_c)^2 over its H*W pixels (fp32, in an order fixed by H*W), [3C] H*W (int32)
 *   backward, first:   1: max |dL/d(fc output)| of the utterance; every rank then uses the loss scale of the union
 *   backward, layer i: 2C: [0,C) sum g_z, [C,2C) sum g_z * xhat (xhat from the global mean / rstd)
 * The statistics combine the records in double around record 0's pivot; dgamma / dbeta are this rank's own sums (the
 * data-parallel gradient reduction adds the ranks'), the BatchNorm input gradient uses the global sums.  Every rank
 * must run the same stages in the same order.  The context works with dsk_train_ctx_read, dsk_train_ctx_commit_stats
 * (dsk_set_defer_running_stats applies at dsk_sync_forward_begin) and dsk_train_ctx_release; dsk_rescnn_backward
 * refuses it.  Calls out of sequence return DSK_ERR_STATE, n_total < B DSK_ERR_INVALID.  x, emb and the gathered
 * buffer must stay alive until the stage's work on `stream` has run. */
int32_t dsk_sync_forward_begin(dsk_handle h, const float* x, int32_t B, int32_t T, float* emb, dsk_train_ctx* ctx,
                               void* stream);
int32_t dsk_sync_backward_begin(dsk_handle h, dsk_train_ctx ctx, const float* grad_emb, const dsk_grads* grads,
                                void* stream);
int32_t dsk_sync_records(dsk_handle h, dsk_train_ctx ctx, void** ptr, int64_t* bytes);
int32_t dsk_sync_stage(dsk_handle h, dsk_train_ctx ctx, const void* gathered, int32_t n_total, int32_t* more,
                       void* stream);

/* Device timing of the next dsk_rescnn_forward calls (which then launch kernel by kernel, not as a graph).
 * enable = 1: CUDA events are recorded on `stream` around every kernel of the forward (order: conv1, the 11
 * tensor-core convs in network order, pool, fc, l2norm); enable = 2: only at the section boundaries
 * conv1 | 11 tensor-core convs | tail (3 values), so the conv chain runs back to back as in production.  dsk_get_launch_times waits for the last profiled forward (the only call in this
 * library that blocks the host) and returns its per-launch milliseconds. Used by bench.py's roofline. */
int32_t dsk_set_profiling(dsk_handle h, int32_t enable);
int32_t dsk_get_launch_times(dsk_handle h, float* ms_out, int32_t cap, int32_t* n_out);

/* One fused conv layer on NHWC 16-bit tensors: out = clip(conv(in, w)*scale + bias (+res)).
 * Building block of dsk_rescnn_forward, exported for unit tests against F.conv2d.
 * ksize/stride in {(3,1),(5,2)}; cin, cout multiples of 64; flags: 1 = add residual, 2 = clip to [0,clip_hi].
 * w_packed comes from dsk_pack_conv_weight. */
int32_t dsk_conv2d_nhwc(dsk_handle h, const void* in, const void* w_packed, const float* scale, const float* bias,
                        const void* res, void* out, int32_t B, int32_t Hin, int32_t Win, int32_t cin, int32_t cout,
                        int32_t ksize, int32_t stride, int32_t flags, float clip_hi, void* stream);
/* Backward building blocks of dsk_rescnn_backward, exported for unit tests against torch autograd.
 * dgrad: g_in (B,Hin,Win,cin) = d/d(input) of conv(input, w) given G (B,Hout,Wout,cout) (+ res, stride 1 only).
 * wgrad: dw (cout,cin,k,k) fp32 = mult * d/d(w) given G and the conv input X (B,Hin,Win,cin). */
int32_t dsk_conv2d_dgrad_nhwc(dsk_handle h, const void* G, const float* w_oihw, const void* res, void* gin, int32_t B,
                              int32_t Hin, int32_t Win, int32_t cin, int32_t cout, int32_t ksize, int32_t stride,
                              void* stream);
int32_t dsk_conv2d_wgrad_nhwc(dsk_handle h, const void* G, const void* X, float* dw_oihw, int32_t B, int32_t Hin,
                              int32_t Win, int32_t cin, int32_t cout, int32_t ksize, int32_t stride, float mult,
                              void* stream);
/* y = clip(BatchNorm_train(raw) (+res), 0, 20) on an NHWC tensor viewed as [M][C] (raw fp32, y/res 16-bit); writes the
 * batch mean / rstd and updates the running statistics (model.py:59,62 in train mode + :79-80). */
int32_t dsk_bn_act_train_forward(dsk_handle h, const float* raw, const float* gamma, const float* beta,
                                 float* running_mean, float* running_var, const void* res, void* y, float* mean,
                                 float* rstd, int64_t M, int32_t C, void* stream);
/* The same with the statistics of the synchronised path: raw holds B utterances of HW pixels each (rows
 * [u*HW, (u+1)*HW) are utterance u); one record per utterance, combined as dsk_sync_stage combines gathered records. */
int32_t dsk_bn_act_sync_train_forward(dsk_handle h, const float* raw, const float* gamma, const float* beta,
                                      float* running_mean, float* running_var, const void* res, void* y, float* mean,
                                      float* rstd, int32_t B, int32_t HW, int32_t C, void* stream);
/* its backward: gy -> G (w.r.t. raw), gres (w.r.t. res, may be NULL), dgamma, dbeta (x inv_scale). */
int32_t dsk_bn_act_train_backward(dsk_handle h, const void* gy, const void* y, const float* raw, const float* gamma,
                                  const float* mean, const float* rstd, void* G, void* gres, float* dgamma,
                                  float* dbeta, int64_t M, int32_t C, float inv_scale, void* stream);
/* The eval forward's convs on the zero-padded NHWC layout with halo reuse (csrc/conv3x3_halo.cuh), exported for
 * unit tests.  Standard padded tensor: [dsk_padded_positions(N,H,W)][C] 16-bit, pixel (n,h,w) at position
 * (n*(H+1)+h+1)*(W+1) + w+1, every other position zero.  Parity-planar tensor of an (N,H,W,C) image (H, W even):
 * four planes p = (h&1)*2 + (w&1), plane p = standard padded tensor of geometry (N, H/2, W/2) holding pixel
 * (n, h>>1, w>>1), planes dsk_padded_positions(N,H/2,W/2) positions apart.  W <= 34.
 * dsk_conv3x3_padded: 3x3 s1 p1, C -> C, standard in; out standard (out_planar = 0) or parity-planar (1).
 * dsk_conv5x5s2_planar: 5x5 s2 p2, parity-planar input of the (N, 2*Hout, 2*Wout, cin) image -> standard padded out. */
int32_t dsk_conv3x3_padded(dsk_handle h, const void* in, const void* w_packed, const float* scale, const float* bias,
                           const void* res, void* out, int32_t N, int32_t H, int32_t W, int32_t C, int32_t flags,
                           float clip_hi, int32_t out_planar, void* stream);
int32_t dsk_conv5x5s2_planar(dsk_handle h, const void* in_planar, const float* w_oihw, const float* scale,
                             const float* bias, void* out, int32_t N, int32_t Hout, int32_t Wout, int32_t cin,
                             int32_t cout, int32_t flags, float clip_hi, void* stream);
int64_t dsk_padded_positions(int32_t N, int32_t H, int32_t W);
/* Debug: device buffer of 3*512 int64 that dsk_conv3x3_padded fills with clock64 stamps of CTA 0
 * (producer / MMA / epilogue roles); NULL switches tracing off. */
int32_t dsk_debug_set_trace(dsk_handle h, void* device_buffer);
/* Debug / test: copies of the intermediate tensors of a train backward, which otherwise live in buffers that the next
 * layer overwrites.  Every non-NULL entry receives, by cudaMemcpyAsync on the backward's stream at the point where the
 * tensor is final, B*H*W*C contiguous values (B, T, C, H, W of the context; layer i as act_shape: C = 64 << i/3,
 * H = T >> (i/3 + 1), W = 64 >> (i/3 + 1); E the embedding size).  S is the backward's loss scale. */
typedef struct {
  void* gy[DSK_NUM_CONV];    /* 16-bit NHWC: gradient w.r.t. layer i's output y_i, times S, as the BatchNorm backward reads it */
  void* G[DSK_NUM_CONV];     /* 16-bit NHWC: gradient w.r.t. the raw conv output raw_i (after the BatchNorm backward), times S */
  void* gres[DSK_NUM_CONV];  /* 16-bit NHWC, i % 3 == 2 only: the skip-branch gradient (gy_i where 0 < y_i < 20, else 0) */
  float* g_fc;               /* (B, E) fp32: the l2-norm backward's output, dL/d(fc output) */
  float* fc_out;             /* (B, E) fp32: the saved fc output the l2-norm backward read */
  float* dP;                 /* (B, 2048) fp32: gradient w.r.t. the pooled fc input, column w*512 + c, before the pool backward */
  float* loss_scale;         /* 2 floats: {S, 1/S} of this backward */
} dsk_backward_capture;
/* Sets (copies *cap) or, with cap == NULL, clears the capture.  It stays set for every following dsk_rescnn_backward and
 * synchronised backward (dsk_sync_backward_begin / dsk_sync_stage) of this handle; the caller keeps the buffers alive.
 * Capturing adds copies only: no kernel and no result changes, and with the capture off the launches are those of a
 * build without it. */
int32_t dsk_debug_set_backward_capture(dsk_handle h, const dsk_backward_capture* cap);
int32_t dsk_pack_conv_weight(dsk_handle h, const float* w_oihw, void* w_packed, int32_t cout, int32_t cin,
                             int32_t ksize, void* stream);
/* fp32 NCHW <-> 16-bit NHWC converters (test helpers; also used at the boundary for C>1 inputs) */
int32_t dsk_nchw_f32_to_nhwc16(dsk_handle h, const float* in, void* out, int32_t B, int32_t C, int32_t H, int32_t W,
                               void* stream);
int32_t dsk_nhwc16_to_nchw_f32(dsk_handle h, const void* in, float* out, int32_t B, int32_t C, int32_t H, int32_t W,
                               void* stream);

/* PairwiseDistance(p=2).forward (reference model.py:8-18): out[i] = sqrt(sum_j (x1-x2)^2 + 1e-4/D). */
int32_t dsk_pairwise_distance(const float* x1, const float* x2, int32_t B, int32_t D, float* out, void* stream);
/* d(out)/d(x1) and d(out)/d(x2) given grad_out (B,), dist (B,) from the forward. Either grad pointer may be NULL. */
int32_t dsk_pairwise_distance_bwd(const float* x1, const float* x2, const float* dist, const float* grad_out,
                                  int32_t B, int32_t D, float* grad_x1, float* grad_x2, void* stream);

/* TripletMarginLoss(margin).forward (reference model.py:19-33):
 * loss = mean(clamp(margin + d_p - d_n, 0)). Writes loss (1,), d_p (B,), d_n (B,).  As torch.clamp, the clamp keeps
 * NaN: a row with a NaN or an infinity gives the reference's non-finite loss (NaN, or +inf for an infinite d_p; an
 * infinite d_n alone clamps to 0).  The backward passes the gradient where the hinge is >= 0, false for NaN. */
int32_t dsk_triplet_loss(const float* a, const float* p, const float* n, int32_t B, int32_t D, float margin,
                         float* loss, float* d_p, float* d_n, void* stream);
/* Gradients of the loss w.r.t. a, p, n scaled by grad_loss (device scalar). */
int32_t dsk_triplet_loss_bwd(const float* a, const float* p, const float* n, const float* d_p, const float* d_n,
                             const float* grad_loss, int32_t B, int32_t D, float margin, float* ga, float* gp,
                             float* gn, void* stream);

/* "Choose the hard negatives" (reference train_triplet.py:251-262):
 * idx = ascending indices i with d_n[i] - d_p[i] < margin  (== np.where(mask == 1)); count on device. */
int32_t dsk_margin_select(const float* d_p, const float* d_n, int32_t B, float margin, int64_t* idx,
                          int32_t* count, void* stream);
/* Row gather out[j] = src[idx[j]] for j < *count (train_triplet.py:265-274), row = row_elems fp32. */
int32_t dsk_gather_rows(const float* src, const int64_t* idx, const int32_t* count, int32_t max_rows,
                        int64_t row_elems, float* out, void* stream);

/* All-pairs distance + per-row k smallest over different-label columns (BASELINE config 4; no reference
 * implementation exists — defined from PairwiseDistance, model.py:13-18):
 * D[i][j] = sqrt(sum_d (E[i]-E[j])^2 + 1e-4/Dim), candidates j with labels[j] != labels[i];
 * ties broken by lower j. Writes idx (N,k) int64 and val (N,k) fp32, ascending distance. */
/* Same result (bit-identical indices and values), computed with a wgmma fp16 Gram GEMM + candidate selection + exact
 * fp32 refinement of the k+8 best candidates per row (exact row scan on the device when the safety margin is not met).
 * Falls back to dsk_allpairs_topk when D % 64 != 0 or k > 8. */
int32_t dsk_allpairs_topk_tc(dsk_handle h, const float* E, const int64_t* labels, int32_t N, int32_t D, int32_t k,
                             int64_t* idx, float* val, void* stream);
int32_t dsk_allpairs_topk(const float* E, const int64_t* labels, int32_t N, int32_t D, int32_t k, int64_t* idx,
                          float* val, void* stream);

/* Batch-hard triplet loss over one batch (P speakers x K utterances; no reference implementation exists - built from
 * PairwiseDistance, model.py:13-18, and the hinge of TripletMarginLoss, model.py:27-33).  d(i,j) is the value
 * dsk_allpairs_topk returns.  Per anchor i: pos_idx = argmax d(i,j) over j != i with labels[j] == labels[i], neg_idx =
 * argmin d(i,j) over labels[j] != labels[i], ties to the lower j; d_ap, d_an those distances (-1 / 0 when there is no
 * positive, -1 / +inf when there is no negative); valid[i] = 1 iff both exist (depends on the labels only).
 * loss (1,) = (1/V) sum over valid i of clamp(margin + d_ap - d_an, 0) in a fixed order, V = #valid; 0 when V = 0.
 * Non-finite rows: a NaN distance is never selected (an infinite one is, with the same tie rule).  An anchor whose row
 * holds a NaN or an infinity gets d_ap = d_an = NaN, keeps the indices of the scans, and is valid iff its label has
 * another row and another label exists: the loss is NaN, and its hinge passes no gradient.
 * h != NULL and D % 64 == 0: the Gram plan of dsk_allpairs_topk_tc (cached in h, fp16 or bf16 per h) with exact fp32
 * refinement; otherwise (h may be NULL) the exact CUDA-core all-pairs matrix.  Both give the same bits.
 * 2 <= N <= DSK_BATCH_HARD_MAX_N (the N x N fp32 distance matrix, 1 GiB at the limit). */
#define DSK_BATCH_HARD_MAX_N 16384
int32_t dsk_batch_hard_triplet(dsk_handle h, const float* E, const int64_t* labels, int32_t N, int32_t D, float margin,
                               float* loss, int64_t* pos_idx, int64_t* neg_idx, float* d_ap, float* d_an,
                               uint8_t* valid, void* stream);
/* Its backward: gE (N,D) = d loss / d E scaled by grad_loss (device scalar), WRITTEN not accumulated.  The hinge passes
 * the gradient where margin + d_ap - d_an >= 0 (torch.clamp); row terms (E_i - E_j) / d(i,j).  Deterministic, no float
 * atomics: row j adds its own anchor term, then the terms of the anchors that chose j, in ascending anchor order. */
int32_t dsk_batch_hard_triplet_bwd(const float* E, const int64_t* pos_idx, const int64_t* neg_idx, const float* d_ap,
                                   const float* d_an, int32_t N, int32_t D, float margin, const float* grad_loss,
                                   const uint8_t* valid, float* gE, void* stream);
/* Row-range form of the batch-hard op, for sharding the anchors of one N-row batch E (e.g. across data-parallel ranks)
 * with results bit-identical to the single-device op on the whole batch.  Rows [row0, row0 + rows) of E are the
 * anchors: 2 <= N <= DSK_BATCH_HARD_MAX_N, 0 <= row0, 1 <= rows, row0 + rows <= N (else DSK_ERR_INVALID).
 * dsk_batch_hard_select_rows: outputs (rows,) hold anchor row0 + i's selection as in dsk_batch_hard_triplet (indices
 * global in [0, N), self-exclusion j != row0 + i, the same tie rules and bits).  h != NULL and D % 64 == 0: the Gram
 * plan is rows_pad x Npad and is cached in h for (N, D, row0, rows); a change of any of them rebuilds it, which
 * synchronises the stream.  dsk_batch_hard_triplet = select_rows(0, N) + dsk_batch_hard_mean.
 * dsk_batch_hard_mean: the loss of dsk_batch_hard_triplet from the selection of all N anchors.
 * dsk_batch_hard_triplet_bwd_rows: rows [row0, row0 + rows) of dsk_batch_hard_triplet_bwd's gE into gE_rows (rows, D);
 * the selection arrays cover all N anchors.  dsk_batch_hard_triplet_bwd = bwd_rows(0, N). */
int32_t dsk_batch_hard_select_rows(dsk_handle h, const float* E, const int64_t* labels, int32_t N, int32_t D,
                                   int32_t row0, int32_t rows, int64_t* pos_idx, int64_t* neg_idx, float* d_ap,
                                   float* d_an, uint8_t* valid, void* stream);
int32_t dsk_batch_hard_mean(const float* d_ap, const float* d_an, const uint8_t* valid, int32_t N, float margin,
                            float* loss, void* stream);
int32_t dsk_batch_hard_triplet_bwd_rows(const float* E, const int64_t* pos_idx, const int64_t* neg_idx,
                                        const float* d_ap, const float* d_an, const uint8_t* valid, int32_t N,
                                        int32_t D, int32_t row0, int32_t rows, float margin, const float* grad_loss,
                                        float* gE_rows, void* stream);

/* Additive angular margin softmax (ArcFace / AAM-softmax) over a cosine classifier (no reference implementation exists;
 * the usual modern form of the reference's softmax over the speaker classifier, train_triplet.py:277-287).  For
 * embeddings E (N,D), class weights W (C,D) (e.g. model.classifier.weight), int64 labels y, margin m >= 0, scale s > 0:
 *   e^_i = e_i / max(||e_i||, 1e-12), w^_c likewise (F.normalize);  cos (N,C) = e^_i . w^_c;
 *   target column: sin = sqrt(clamp(1 - cos^2, 0, 1)), phi = cos > cos(pi - m) ? cos cos m - sin sin m
 *                                                                           : cos - sin(pi - m) m;
 *   logit_ic = s * (c == y_i ? phi : cos);  lse (N,) = logsumexp_c logit_ic;
 *   loss (1,) = (1/N) sum_i (lse_i - logit_{i,y_i}), summed in a fixed order.  A label outside [0, C) yields NaN.
 * cos and lse are caller-owned outputs that dsk_aam_softmax_bwd reads.  The cosines run on the tensor cores in fp16
 * (whatever the handle's operand type) with each operand split into hi + lo halves, which keeps them at fp32-level
 * accuracy; the target column's cosine is recomputed in fp64.  Every row of cos, lse and gE depends only on that row's
 * embedding and label (and W): sharding the batch
 * over ranks gives bit-identical rows when grad_loss / N is the same.
 * The GEMM plan and its operand buffers are cached in h for (N, C, D), in a slot of their own; a change rebuilds them,
 * which synchronises the stream.  1 <= N, 2 <= C <= DSK_AAM_MAX_C, D % 64 == 0, else DSK_ERR_INVALID. */
#define DSK_AAM_MAX_C 65536
int32_t dsk_aam_softmax(dsk_handle h, const float* E, const float* W, const int64_t* labels, int32_t N, int32_t C,
                        int32_t D, float margin, float scale, float* loss, float* cos, float* lse, void* stream);
/* Its backward: gE (N,D) and gW (C,D) = d loss / d E, d loss / d W scaled by grad_loss (device scalar), WRITTEN not
 * accumulated.  dcos = s (softmax - onehot) grad_loss / N, times d phi / d cos on the target column (cos m + sin m
 * cos / sin; cos m at sin = 0; 1 below cos(pi - m)), then gE^ = dcos W^, gW^ = dcos^T E^ and the F.normalize Jacobians
 * g_i = (g^_i - e^_i (e^_i . g^_i)) / max(||e_i||, 1e-12).  Deterministic: no float atomics; the two GEMMs split K
 * into fixed slices of 512 classes / utterances whose outputs are added in slice order. */
int32_t dsk_aam_softmax_bwd(dsk_handle h, const float* E, const float* W, const int64_t* labels, const float* cos,
                            const float* lse, int32_t N, int32_t C, int32_t D, float margin, float scale,
                            const float* grad_loss, float* gE, float* gW, void* stream);

/* Generalised end-to-end (GE2E) loss against in-batch speaker centroids (Wan et al., ICASSP 2018; no reference
 * implementation exists).  For embeddings E (N,D) and a batch of P speakers given as a CSR: speaker k's rows are
 * S_k = order[offsets[k] .. offsets[k+1]) (n_k of them, ascending row index within a speaker), col[i] = the speaker of
 * row i (device int64; the host builds them from the labels, speakers in ascending label order):
 *   e^_i = e_i / max(||e_i||, 1e-12) (F.normalize);  inclusive centroid c_k = (1/n_k) sum_{u in S_k} e^_u (exactly
 *   dsk_class_centroids);  exclusive centroid c_k^(-i) = (1/(n_k - 1)) sum_{u in S_k, u != i} e^_u (n_k >= 2);
 *   c^ = c / max(||c||, 1e-12);  cos (N,P): cos_ik = e^_i . c^_k for k != y_i, cos_{i,y_i} = e^_i . c^_{y_i}^(-i)
 *   (a row of a singleton speaker keeps the inclusive cosine there);  S_ik = max(w, 1e-6) cos_ik + b.
 *   Row i is valid when n_{y_i} >= 2 (with P >= 2); V = the number of valid rows.  Row losses:
 *     DSK_GE2E_SOFTMAX:  L_i = logsumexp_k S_ik - S_{i,y_i};                       rec[i] = logsumexp_k S_ik
 *     DSK_GE2E_CONTRAST: L_i = 1 - sigmoid(S_{i,y_i}) + max_{k != y_i} sigmoid(S_ik);  rec[i] = that k, ties to the
 *                        lowest column (an integer stored in fp32)
 *   loss (1,) = (1/V) sum over valid i of L_i, summed in a fixed order.  A singleton speaker's row has no loss term,
 *   but its centroid is a column of every other row.
 * w and b are device scalars (nothing is read back); cos and rec are caller-owned outputs that dsk_ge2e_bwd reads.
 * Accuracy: the non-target cosines run on the AAM-softmax op's hi/lo fp16 tensor-core GEMM against the centroids
 * (computed in fp64, rounded to fp32), within ~1e-6 of fp64; the target cosine is computed in fp64 from the fp32 rows
 * in CSR order and rounded once.
 * The GEMM plan and its buffers are cached in h for (N, P, D), in a slot of their own (the AAM, scoring, search and
 * all-pairs plans are untouched); a change rebuilds them, which synchronises the stream.  Cost beyond the GEMMs:
 * O(sum_k n_k^2 D) for the exclusive centroids.
 * 2 <= P <= DSK_AAM_MAX_C, D % 64 == 0, 1 <= V <= N, method one of the two below, else DSK_ERR_INVALID before any
 * launch. */
#define DSK_GE2E_SOFTMAX 0
#define DSK_GE2E_CONTRAST 1
int32_t dsk_ge2e(dsk_handle h, const float* E, int32_t N, int32_t D, const int64_t* order, const int64_t* offsets,
                 const int64_t* col, int32_t P, int32_t V, const float* w, const float* b, int32_t method, float* loss,
                 float* cos, float* rec, void* stream);
/* Its backward: gE (N,D), gw (1,), gb (1,) = d loss / d (E, w, b) scaled by grad_loss (device scalar), WRITTEN not
 * accumulated.  dS_ik = grad_loss / V * dL_i / dS_ik on valid rows and 0 elsewhere, dcos = max(w, 1e-6) dS;
 * gw = sum dS cos over every entry where w >= 1e-6 (torch.clamp passes the gradient there), else 0; gb = sum dS for
 * contrast, and EXACTLY 0 for softmax: b cancels out of the softmax loss, and the rounding residue torch autograd
 * returns instead would be amplified by an adaptive optimizer into steps of size lr.  gw and gb are summed in fp64 in a
 * fixed order.  In e^-space, g^_i is the sum of
 *   the direct term       sum_{k != y_i} dcos_ik c^_k + dcos_{i,y_i} c^_{y_i}^(-i);
 *   the inclusive terms   g^c_k = sum_{i: y_i != k} dcos_ik e^_i, gc_k = (g^c_k - c^_k (c^_k . g^c_k)) / max(||c_k||,
 *                         1e-12), added as gc_k / n_k to every member of S_k;
 *   the exclusive terms   for every valid row j of speaker k, the Jacobian at c_k^(-j) applied to dcos_{j,k} e^_j,
 *                         divided by n_k - 1 and added to every member u != j of S_k, in ascending j;
 * then gE_u = (g^_u - e^_u (e^_u . g^_u)) / max(||e_u||, 1e-12).  The two products run on the AAM plan's GEMMs in
 * fixed K slices; the exclusive-centroid terms are computed in fp64 from the fp32 rows, as fixed-order sums over each
 * speaker's members.  Deterministic: no float atomics, two calls give the same bits. */
int32_t dsk_ge2e_bwd(dsk_handle h, const float* E, int32_t N, int32_t D, const int64_t* order, const int64_t* offsets,
                     const int64_t* col, int32_t P, int32_t V, const float* w, const float* b, int32_t method,
                     const float* cos, const float* rec, const float* grad_loss, float* gE, float* gw, float* gb,
                     void* stream);
/* Row-range form of the GE2E op, for sharding the rows of one N-row batch E (e.g. across data-parallel ranks, each
 * holding the gathered E) with results bit-identical to the whole-batch op.  The centroids, the exclusive centroid of
 * every row and the fp64 row norms always come from all N rows, so a speaker's rows may sit anywhere in the batch.
 * 0 <= row0, 1 <= rows, row0 + rows <= N, plus the limits of dsk_ge2e, else DSK_ERR_INVALID before any launch.
 * The plan is cached in h for (N, P, D, row0, rows), in the GE2E slot; a change rebuilds it, which synchronises the
 * stream.  dsk_ge2e = rows(0, N) + dsk_ge2e_mean;  dsk_ge2e_bwd = dcos_rows(0, N) + bwd_rows(0, N).
 * dsk_ge2e_rows: rows [row0, row0 + rows) of dsk_ge2e's cos and rec into cos (rows, P) and rec (rows,), and the rows'
 *   loss terms L_i (0 on invalid rows) into row_loss (rows,).  The cosine GEMM runs only for the rows x P block.
 * dsk_ge2e_mean: dsk_ge2e's loss from row_loss (N,) of all N rows: (1/V) sum_i row_loss[i] in a fixed order.
 * dsk_ge2e_dcos_rows: for the range, from its cos and rec (rows, P) / (rows,) and the whole batch's CSR: dcos (rows, P)
 *   = max(w, 1e-6) dS as in dsk_ge2e_bwd, with the target column zeroed and its value in tdc (rows,); gw and gb (1,)
 *   are the range's shares of dsk_ge2e_bwd's gw and gb (fp64 sums over the range's rows in a fixed order, rounded
 *   once; gb exactly 0 for softmax).  Summed over the ranges of a split they equal the whole op's to ~1e-7 relative.
 * dsk_ge2e_bwd_rows: rows [row0, row0 + rows) of dsk_ge2e_bwd's gE into gE_rows (rows, D), from dcos (N, P) and tdc
 *   (N,) of ALL N rows (the concatenation of every range's dsk_ge2e_dcos_rows).  gC^ = dcos^T E^ runs over all N rows
 *   in the whole op's K slices, the exclusive-centroid terms for the members of every speaker with a row in the range,
 *   and gE^ = dcos C^ only for the rows x P block. */
int32_t dsk_ge2e_rows(dsk_handle h, const float* E, int32_t N, int32_t D, const int64_t* order, const int64_t* offsets,
                      const int64_t* col, int32_t P, int32_t V, const float* w, const float* b, int32_t method,
                      int32_t row0, int32_t rows, float* cos, float* rec, float* row_loss, void* stream);
int32_t dsk_ge2e_mean(const float* row_loss, int32_t N, int32_t V, float* loss, void* stream);
int32_t dsk_ge2e_dcos_rows(const float* cos, const float* rec, int32_t N, const int64_t* offsets, const int64_t* col,
                           int32_t P, int32_t V, const float* w, const float* b, int32_t method, const float* grad_loss,
                           int32_t row0, int32_t rows, float* dcos, float* tdc, float* gw, float* gb, void* stream);
int32_t dsk_ge2e_bwd_rows(dsk_handle h, const float* E, int32_t N, int32_t D, const int64_t* order,
                          const int64_t* offsets, const int64_t* col, int32_t P, const float* dcos, const float* tdc,
                          int32_t row0, int32_t rows, float* gE_rows, void* stream);

/* Cosine scoring of verification trials with adaptive symmetric score normalisation (AS-norm) against an impostor
 * cohort (no reference implementation exists; the reference scores Euclidean distances, eval_metrics.py:5-50).  Rows are
 * normalised as in F.normalize, x^ = x / max(||x||, 1e-12).
 *   dsk_cosine_matrix: cos (M,Nc) = a^_i . b^_j for A (M,D) and B (Nc,D), fp32 out.
 *   dsk_topk_mean_std: for every row r of S (rows x cols, row stride ld floats), tau = its k-th largest value and the
 *     multiset of every value > tau plus as many copies of tau as make k values (independent of tie breaking);
 *     mean[r] = its mean, std[r] = its standard deviation with divisor k - 1 (torch.std), both accumulated in fp64 in a
 *     fixed order as two passes (mean, then sum (x - mean)^2) and rounded to fp32.  A row with a NaN gives NaN for both;
 *     +-inf and +-0 are ordered as numbers.  One CTA per row: an exact radix select of tau on order-preserving uint32
 *     keys (shared-memory histograms), the row staged in shared memory when cols <= 16384.  No float atomics.
 *   dsk_cohort_stats: mean, std (M,) of the k largest cosines of each row of E (M,D) against the cohort (Nc,D) (k = Nc:
 *     plain S-norm); bit-identical to dsk_topk_mean_std(dsk_cosine_matrix(E, cohort)).
 * The cosines run on the tensor cores as the AAM-softmax op's do (fp16 whatever the handle's type, each operand split
 * into hi + lo halves, K = 3D).  E is processed in row chunks: rows per chunk = the largest multiple of 128 with
 * chunk x Npad x 4 B <= 256 MiB (Npad = Nc rounded up to 128), at least 128, and no more than M rounded up to 128.
 * Every chunk reuses one operand buffer and one set of GEMM launches in stream order, and each row's outputs depend only
 * on that row and the cohort: they are bit-identical whatever M, wherever the row sits and however E is split.  The
 * plan is cached in h for (Nc, D, chunk), in a slot of its own (the all-pairs, batch-hard and AAM plans are untouched);
 * a change rebuilds it, which synchronises the stream.  The cohort's operand image is rebuilt on every call.
 * M >= 1, 2 <= Nc <= DSK_SCORE_MAX_COHORT, 2 <= k <= Nc, D % 64 == 0, else DSK_ERR_INVALID. */
#define DSK_SCORE_MAX_COHORT 65536
int32_t dsk_cosine_matrix(dsk_handle h, const float* A, int32_t M, const float* B, int32_t Nc, int32_t D, float* cos,
                          void* stream);
int32_t dsk_topk_mean_std(const float* S, int32_t rows, int32_t cols, int64_t ld, int32_t k, float* mean, float* std,
                          void* stream);
int32_t dsk_cohort_stats(dsk_handle h, const float* E, int32_t M, const float* cohort, int32_t Nc, int32_t D,
                         int32_t k, float* mean, float* std, void* stream);
/* Trial scores: trials (T,2) int64 (e, t) index rows of one embedding table X (U,D).  raw[i] = x^_e . x^_t in fp64 from
 * the fp32 inputs, rounded to fp32; with mean / std (U,) given (dsk_cohort_stats of X), normed[i] = 0.5 ((s - mean_e) /
 * std_e + (s - mean_t) / std_t) in fp64 from the unrounded s (AS-norm; std = 0 gives what IEEE division gives).  mean and
 * std may both be NULL, and then normed is not written.  An index outside [0, U) gives NaN in both outputs and reads
 * nothing.  One warp per trial, fixed order. */
int32_t dsk_score_trials(const float* X, int32_t U, int32_t D, const int64_t* trials, int64_t T, const float* mean,
                         const float* std, float* raw, float* normed, void* stream);

/* Speaker identification: exact top-k cosine search against an enrolled gallery of any size (no reference
 * implementation exists).  The search order ranks a above b when a > b as numbers, ties going to the lower column;
 * -0 == +0, and NaN ranks below every number (-inf included), so one corrupt gallery row never becomes every query's
 * top-1.  idx / val are (rows, k) row-major: the k first columns of each row in that order and their values (the
 * input's bits).
 *   dsk_topk_indices: the search order over every row r of S (rows x cols, row stride ld floats).  One CTA per row: the
 *     k-th key by the exact radix select of dsk_topk_mean_std, every column above it plus the lowest columns equal to
 *     it (an ordered compaction), a bitonic sort of the k entries in shared memory.  The row is staged in shared memory
 *     when cols <= 16384.  1 <= k <= min(cols, DSK_SEARCH_MAX_K), cols <= DSK_SCORE_MAX_COHORT, ld >= cols.
 *   dsk_cosine_topk: the search order over the row of cosines of query i of Q (M,D) against the gallery G (Ng,D), for
 *     any Ng >= k.  val is exactly the fp32 cosine dsk_cosine_matrix gives for that pair, so the result equals
 *     dsk_topk_indices of dsk_cosine_matrix(Q, G) for Ng <= DSK_SCORE_MAX_COHORT, and of dsk_cosine_matrix of column
 *     slices, concatenated, beyond.  The gallery is taken in column chunks of 16384 rows in ascending order, each with
 *     its operand image built once; the queries in row chunks as in dsk_cohort_stats (Npad = 16384, or Ng rounded up to
 *     128 for a smaller gallery).  Each chunk's k best are merged into idx / val, which hold the running lists; the
 *     workspace is one row chunk x k entries (stream-ordered allocation).  A query's result depends only on that query
 *     and G: bit-identical whatever M and wherever the row sits.  The plan is cached in h in a slot of its own (the
 *     scoring, all-pairs, batch-hard and AAM plans are untouched); a change rebuilds it, which synchronises the stream.
 *     M >= 1, 1 <= k <= DSK_SEARCH_MAX_K, Ng >= k, D % 64 == 0.
 *   dsk_class_centroids: enrolment.  out[s] (S,D) = (1/n_s) * the sum of x^_u over u = order[offsets[s] ..
 *     offsets[s+1]), with x^_u = X[u] / max(||X[u]||, 1e-12) in fp64 from the fp32 row, summed in fp64 in that order
 *     and rounded to fp32; n_s = offsets[s+1] - offsets[s].  An empty segment gives a zero row, an index outside [0, U)
 *     a NaN row.  One CTA per class and 256 columns, no float atomics.  order, offsets (S+1) are device int64.
 * Arguments outside these limits return DSK_ERR_INVALID. */
#define DSK_SEARCH_MAX_K 1024
int32_t dsk_topk_indices(const float* S, int32_t rows, int32_t cols, int64_t ld, int32_t k, int64_t* idx, float* val,
                         void* stream);
int32_t dsk_cosine_topk(dsk_handle h, const float* Q, int32_t M, const float* G, int32_t Ng, int32_t D, int32_t k,
                        int64_t* idx, float* val, void* stream);
int32_t dsk_class_centroids(const float* X, int32_t U, int32_t D, const int64_t* order, const int64_t* offsets,
                            int32_t S, float* out, void* stream);

/* Diarization: agglomerative hierarchical clustering of N items from their similarities (no reference implementation
 * exists).  S (N x N fp32, device, row stride ld floats) holds similarities, higher meaning closer; only its strict upper
 * triangle is read (the diagonal and the lower triangle may hold anything).  The distance is d_ij = 1 - (double)S[i][j]
 * for i < j, rounded once in fp64 (numpy's 1.0 - S.astype(float64)).  A non-finite value in the upper triangle gives
 * DSK_ERR_INVALID after one validation pass and one flag read.
 *   Linkage: DSK_LINKAGE_AVERAGE (UPGMA) or DSK_LINKAGE_COMPLETE, on an fp64 working matrix on the device kept exactly
 *     symmetric.  Merging A u B against C u D (D absent, n_D = 0, when C did not merge in the same round), average is
 *     (nA nC dAC + nA nD dAD + nB nC dBC + nB nD dBD) / ((nA + nB)(nC + nD)) summed in that order, A and C the lower
 *     representatives (a cluster's representative is its smallest original index); complete is the max of the same.
 *   Rounds (RAC, Sumengen et al. 2021): every live cluster finds its nearest live cluster (ties to the smaller
 *     representative); every mutual pair whose height is <= stop_height merges; the merged rows and columns are
 *     updated; once the live count falls below half the stored dimension the matrix is repacked into a smaller buffer.
 *     For these reducible linkages the dendrogram is the sequential algorithm's.  The rounds run until one cluster is
 *     left or no mutual pair lies at or below stop_height; the cut at stop_k clusters is then taken from the sorted
 *     tree (its first N - stop_k rows), which is exact.  Stopping the rounds at stop_k clusters would not be: a round
 *     may merge a mutual pair far above merges that later rounds make.  The host reads a device-side done flag once per
 *     64 rounds; after it is set the kernels of the batch return at once.
 *   Outputs (host memory; the call synchronises the stream): Z (n_merges, 4) fp64 row-major in scipy's linkage format
 *     [id_a, id_b, height, size], id_a < id_b, points 0..N-1 and the cluster made by row r numbered N + r, rows sorted
 *     by (height, round, representative); with stop_k = 1 and stop_height = +inf the full tree (n_merges = N - 1),
 *     otherwise the first n_merges = min(N - stop_k, merges at or below stop_height) rows of it.  Z must hold N - 1 rows.  labels (N,) int32: the flat clusters at the
 *     stop point, numbered from 0 in the order of each cluster's smallest member.  n_rounds (may be NULL): the rounds
 *     that merged.
 *   Workspace: N^2 + ceil(N/2)^2 doubles and O(N) more, stream-ordered (cudaMallocAsync / cudaFreeAsync).  Index
 *   arithmetic is 64-bit.  2 <= N <= DSK_AHC_MAX_N, ld >= N, 1 <= stop_k <= N, a known linkage, stop_height not NaN,
 *   non-null S, Z, n_merges, labels; else DSK_ERR_INVALID. */
#define DSK_AHC_MAX_N 32768
#define DSK_LINKAGE_AVERAGE 0
#define DSK_LINKAGE_COMPLETE 1
int32_t dsk_ahc(const float* S, int32_t N, int64_t ld, int32_t linkage, int32_t stop_k, double stop_height, double* Z,
                int32_t* n_merges, int32_t* labels, int32_t* n_rounds, void* stream);

/* nn.Linear of DeepSpeakerModel.forward_classifier (reference model.py:167,220-223): y (M,N) = x (M,K) w(N,K)^T + b.
 * fp32 on the CUDA cores, fixed summation order (deterministic).  b may be NULL. */
int32_t dsk_linear_forward(const float* x, const float* w, const float* b, int32_t M, int32_t N, int32_t K, float* y,
                           void* stream);
/* its backward: gx (M,K) = gy w, gw (N,K) = gy^T x, gb (N) = column sums of gy; any output pointer may be NULL. */
int32_t dsk_linear_backward(const float* x, const float* w, const float* gy, int32_t M, int32_t N, int32_t K, float* gx,
                            float* gw, float* gb, void* stream);
/* nn.CrossEntropyLoss() over (M,C) logits and int64 labels (reference train_triplet.py:281-285):
 * loss (1,) = mean_i (logsumexp_j logits[i] - logits[i][label_i]); also writes lse (M,) and row_loss (M,) (workspace
 * the backward reads).  A label outside [0,C) yields a NaN row loss, so a NaN loss; the other rows are unaffected. */
int32_t dsk_cross_entropy(const float* logits, const int64_t* labels, int32_t M, int32_t C, float* loss, float* lse,
                          float* row_loss, void* stream);
/* dlogits (M,C) = (softmax(logits) - onehot(labels)) * grad_loss / M; grad_loss is a device scalar.  The row of a
 * label outside [0,C) is all NaN, so an invalid example cannot train the parameters silently. */
int32_t dsk_cross_entropy_bwd(const float* logits, const int64_t* labels, const float* lse, const float* grad_loss,
                              int32_t M, int32_t C, float* dlogits, void* stream);

/* torch.optim.Adagrad step (reference train_triplet.py:369-383, called at :224,291) on ONE flat bucket of n fp32
 * elements (parameters, gradients and the running sum of squares laid out identically), fused with the gradient scale
 * that follows the data-parallel allreduce.  Per element, each step rounded to fp32:
 *   g = grad / grad_div                        (skipped when grad_div == 1; grad_div > 0, e.g. the world size)
 *   g = g / max(*grad_denom, 1e-30)            (only if grad_denom is non-NULL, a device scalar; NaN propagates)
 *   g = fma(p, weight_decay, g)                (skipped when weight_decay == 0)
 *   sum = fma(g, g, sum);  p = p + (g * -clr) / (sqrt(sum) + eps)
 * where -clr = -lr / (1 + (step-1) lr_decay) is computed in double and rounded once to fp32.
 * `step` counts from 1.  After the divisions this is the operation order of torch's foreach Adagrad on CUDA: the
 * result is bit-identical to torch.optim.Adagrad stepping on grad.div(d) with d a CUDA tensor (a true division; ATen
 * turns division by a CPU scalar into a product with its reciprocal).  Buffers must be 16-byte aligned. */
int32_t dsk_adagrad_step(float* param, const float* grad, float* state_sum, int64_t n, double lr, double lr_decay,
                         double weight_decay, double eps, int64_t step, float grad_div, const float* grad_denom,
                         void* stream);

/* Serving pipeline for the reference's test() loop (reference train_triplet.py:337-350: batch to the GPU, model(x),
 * result back - serialised on one stream there).  `primary` owns the weights (dsk_load_weights); the pipeline adds
 * `lanes` handles that borrow them (dsk_share_weights; `primary` stays free for its caller), one compute stream per lane and two copy streams, and keeps depth*lanes device
 * slots.  dsk_pipeline_submit queues, without blocking the host: H2D of the PINNED input batch (B,1,T,64) fp32 -> eval forward
 * on the next lane -> D2H of the (B,E) embeddings into the PINNED output; *ticket identifies the batch.  Both host buffers
 * are accessed asynchronously: leave x_host / emb_host alone until dsk_pipeline_wait(ticket) (blocks the host until that
 * batch's output is complete) or dsk_pipeline_sync.
 * dsk_pipeline_submit_device runs device-resident batches through the same lanes (inputs ordered after `after_stream`);
 * dsk_pipeline_join makes `stream` wait for everything submitted so far; dsk_pipeline_lane_stream returns the cudaStream_t of
 * compute lane 0..lanes-1 (-1: the H2D copy stream, -2: the D2H copy stream) for event timing.  One thread drives a pipeline. */
int32_t dsk_pipeline_create(dsk_pipeline* out, dsk_handle primary, int32_t lanes, int32_t depth);
int32_t dsk_pipeline_destroy(dsk_pipeline p);
int32_t dsk_pipeline_submit(dsk_pipeline p, const float* x_host, int32_t B, int32_t T, float* emb_host, int64_t* ticket);
int32_t dsk_pipeline_submit_device(dsk_pipeline p, const float* x_dev, int32_t B, int32_t T, float* emb_dev, void* after_stream,
                                   int64_t* ticket);
int32_t dsk_pipeline_join(dsk_pipeline p, void* stream);
int32_t dsk_pipeline_wait(dsk_pipeline p, int64_t ticket);
int32_t dsk_pipeline_sync(dsk_pipeline p);
int32_t dsk_pipeline_lane_stream(dsk_pipeline p, int32_t lane, void** stream_out);

/* Log mel-filterbank front-end of the reference (reference audio_processing.py:9-36 mk_MFB with constants.py:
 * python_speech_features.fbank(audio, samplerate, nfilt=64, winlen=0.025) -> 20*log10(max(., 1e-5)) (log_scale) -> minus the
 * per-bin mean over the utterance (subtract_mean, normalize_frames with Scale=False).  audio: n_samples fp32 mono on the
 * device; feat: (dsk_fbank_num_frames(n_samples, sample_rate), 64) fp32 row-major, the (T, 64) layout the network's input
 * is cropped from.  python_speech_features is not vendored in the reference (parity against it unpinned): its published
 * algorithm is restated (pre-emphasis 0.97, 25 ms / 10 ms rectangular frames, NFFT 512, |rfft|^2 / NFFT, triangular mel
 * filters, zeros -> eps).  A NaN or infinite sample makes every frame whose pre-emphasised window covers it (the
 * sample and the next) NaN in all 64 filters, log floor included, as numpy.maximum does; with subtract_mean the
 * utterance's mean, so all its features, are NaN.  This holds for dsk_fbank_batch (the other utterances keep their
 * bits) and dsk_fbank_segments (so an example dsk_wave_augment made NaN is all NaN). */
int64_t dsk_fbank_num_frames(int64_t n_samples, int32_t sample_rate);
int32_t dsk_fbank(const float* audio, int64_t n_samples, int32_t sample_rate, int32_t log_scale, int32_t subtract_mean,
                  float* feat, void* stream);

/* Batched log-fbank and the crops of a feature bank.
 *   dsk_fbank_frame_offsets: host only.  frame_off (U+1) int64 from sample_off (U+1) int64: frame_off[0] = 0,
 *     frame_off[u+1] = frame_off[u] + dsk_fbank_num_frames(sample_off[u+1] - sample_off[u], sample_rate).  Every length
 *     must lie in [1, 2^31) and sample_off[0] >= 0; otherwise DSK_ERR_INVALID.
 *   dsk_fbank_batch: U waveforms, utterance u = audio[sample_off[u] .. sample_off[u+1]) (sample_off on the HOST, int64:
 *     the concatenation may exceed 2^31 samples, each utterance may not) -> feat (frame_off[U], 64) fp32, rows
 *     frame_off[u] .. frame_off[u+1] those of utterance u.  The rows of utterance u are bit-identical to dsk_fbank on
 *     that waveform alone, whatever the other utterances and their order: each utterance starts on a 4-frame block
 *     boundary and its mean is its own block partials added in block order in double.  The filterbank is built and
 *     uploaded once per call; one host synchronisation per call, whatever U.  dsk_fbank is the U = 1 call of it.
 *   dsk_fbank_crops: out (B, 1, T, 64) fp32 from a bank feat (F, 64) fp32 with frame offsets frame_off (U+1) (device
 *     int64): for crop b with u = utt[b], s = start[b], n = frame_off[u+1] - frame_off[u],
 *       out[b, 0, t, m] = feat[frame_off[u] + (s + t) mod n, m]   (wrapping repeats an utterance shorter than T),
 *     set to 0 where t lies in one of the crop's n_time time masks or m in one of its n_freq frequency masks
 *     (time_masks (B, n_time, 2), freq_masks (B, n_freq, 2) device int32 (start, width) pairs: [start, start + width)
 *     clipped to the crop, width 0 = no mask).  u outside [0, U) or s outside [0, n): the whole crop is NaN and nothing
 *     outside feat is read; the other crops are unaffected.  utt, start: device int64 (B,).  One launch, 16-byte
 *     accesses (feat and out 16-byte aligned), no atomics, no host synchronisation. */
int32_t dsk_fbank_frame_offsets(const int64_t* sample_off, int32_t U, int32_t sample_rate, int64_t* frame_off);
int32_t dsk_fbank_batch(const float* audio, const int64_t* sample_off, int32_t U, int32_t sample_rate, int32_t log_scale,
                        int32_t subtract_mean, float* feat, void* stream);
int32_t dsk_fbank_crops(const float* feat, const int64_t* frame_off, int32_t U, const int64_t* utt, const int64_t* start,
                        int32_t B, int32_t T, const int32_t* time_masks, int32_t n_time, const int32_t* freq_masks,
                        int32_t n_freq, float* out, void* stream);

/* Frame-energy voice activity detection (a restatement of the rule of Kaldi's compute-vad, the energy VAD of the usual
 * speaker-embedding recipes) and the runs of kept frames of a feature bank.
 *   Frame energy: E_f = pspec[f][0] + pspec[f][1] + ... + pspec[f][256], added in fp32 in bin order, where pspec is the
 *     power spectrum the fbank computes for frame f (|rfft|^2 / 512 of the pre-emphasised, zero-padded rectangular
 *     frame); 0 is replaced by 2.220446049250313e-16.  This is python_speech_features' `energy` output (the reference's
 *     fbank call returns it and mk_MFB drops it).  Energy row f is feature row f.
 *   Decision, per utterance u of n_u frames: e_f = ln(E_f) in fp64; thr_u = energy_threshold + mean_scale * (S_u / n_u),
 *     S_u the sum of e_f over 4-frame blocks in frame order, the block sums added in block order (independent of the
 *     batch's other utterances); frame f is speech iff #{g in [max(0, f - c), min(n_u - 1, f + c)] : e_g > thr_u} >=
 *     proportion * (the size of that window), c = context.  Recipe values: mean_scale 0.5, context 2, proportion 0.12,
 *     energy_threshold 5.5 - 0.5 ln(2^31) (Kaldi's 5.5 moved from an int16-scale sum of squares of the frame to float
 *     samples and the half-spectrum energy; pre-emphasis not corrected for).  That threshold is not calibrated on
 *     labelled speech.  Cost per frame: min(2c + 1, n_u) comparisons.
 *   dsk_fbank_batch_vad: dsk_fbank_batch (feat bit-identical to it: dsk_fbank_batch is the same host code without the
 *     VAD) plus energy (F,) fp32 (may be NULL) and speech (F,) uint8 0/1, device, F = frame_off[U].  Every utterance's
 *     energies and decisions are bit-identical whatever the batch's other utterances and their order.  One host
 *     synchronisation per call.  Non-finite energy_threshold, mean_scale or proportion, context < 0 or proportion < 0:
 *     DSK_ERR_INVALID.
 *   dsk_frame_runs: the runs of kept frames (mask[row] != 0, mask (F,) uint8 device over the rows of a bank with device
 *     frame offsets frame_off (U+1)) of the K listed utterances utt (device int64, each in [0, U)); list_off (device,
 *     K + 1) holds the prefix sums of their frame counts and P = list_off[K] (host).  runs (capacity, 3) int64 device:
 *     row r = (j, first, end), local frames [first, end) of utterance utt[j], in list order and frame order within an
 *     utterance; a run never spans two utterances.  run_off (capacity + 1) int64 device: the kept frames before run r,
 *     run_off[n_runs] = all kept frames (the offsets of the bank of the runs).  counts (host, 2) = (n_runs, kept frames):
 *     the call's one host read.  Ordered stream compaction (per-tile counts, one fixed-order scan, then the writes), no
 *     atomics.  n_runs > capacity: DSK_ERR_INVALID and no row past capacity is written (the runs of an utterance of n
 *     frames are at most ceil(n / 2)).
 *   dsk_gather_runs: out (rows, 64) fp32, rows = run_off[n_runs] (host): rows run_off[r] .. run_off[r + 1] are bank rows
 *     frame_off[utt[j]] + first .. + end of run r.  16-byte loads and stores (feat, out 16-byte aligned), no host
 *     synchronisation.
 *   Index arithmetic is 64-bit throughout. */
int32_t dsk_fbank_batch_vad(const float* audio, const int64_t* sample_off, int32_t U, int32_t sample_rate,
                            int32_t log_scale, int32_t subtract_mean, double energy_threshold, double mean_scale,
                            int32_t context, double proportion, float* feat, float* energy, uint8_t* speech,
                            void* stream);
int32_t dsk_frame_runs(const uint8_t* mask, const int64_t* frame_off, int32_t U, const int64_t* utt,
                       const int64_t* list_off, int32_t K, int64_t P, int64_t capacity, int64_t* runs, int64_t* run_off,
                       int64_t* counts, void* stream);
int32_t dsk_gather_runs(const float* feat, const int64_t* frame_off, int32_t U, const int64_t* utt, const int64_t* runs,
                        const int64_t* run_off, int64_t n_runs, int64_t rows, float* out, void* stream);

/* Waveform augmentation of training segments (reverberation by room impulse responses and additive noise, the MUSAN +
 * RIR recipe) and the features of equal-length segments.
 *   dsk_fbank_filterbank: host only.  fb[64][257] fp32, the triangular mel filterbank dsk_fbank_batch applies
 *     (python_speech_features get_filterbanks(nfilt=64, nfft=512, samplerate)).
 *   dsk_wave_augment: out (B, L) fp32.  For example b, u = utt[b]:
 *     segment      s[i] = speech[speech_off[u] + (start[b] + i) mod n_u] * 2^-15, i in [0, L)  (n_u = the utterance's
 *                  sample count; int16 PCM, so exactly what librosa.load returns for a 16-bit file; the wrap is crops')
 *     reverb       rir_idx[b] = -1 (or rir_idx NULL): r = s, bit for bit.  Otherwise h = RIR rir_idx[b] (rir[rir_off[i] ..
 *                  rir_off[i+1]), L_h taps, used exactly as stored) and r[i] = sum_{k=0}^{min(i, L_h-1)} h[k] s[i-k]: the
 *                  full convolution truncated to its first L samples, no alignment to the direct path.  Computed by
 *                  uniformly partitioned overlap-save (1024-sample partitions, 2048-point fp32 FFTs, the partitions
 *                  summed in a fixed order).
 *     noise        M <= DSK_AUG_MAX_SOURCES sources per example, (B, M) noise_idx (-1 = none), noise_start, snr_db
 *                  (fp64); n_j is read from the noise bank like s, wrapping.  P(x) = sum x^2 / L in fp64 in a fixed order;
 *                  g_j = sqrt(P(r) / (P(n_j) 10^(snr_j / 10))), 0 when P(n_j) = 0; out[i] = r[i] + sum_j g_j n_j[i]
 *                  evaluated in fp64 and rounded once to fp32.
 *     An index or start outside its bank, a RIR longer than max_rir_len, a noise index < -1 or a non-finite SNR of a
 *     used source makes example b NaN; nothing outside any bank is read and the other examples are unaffected.  Each
 *     example's output depends only on its own arguments (bit-identical for any B, batch position or interleaved call).
 *     Banks (speech / rir / noise samples and their int64 offsets) may be device memory or page-locked host memory (read
 *     over the bus by the same kernels); pageable memory is rejected.  utt, start, rir_idx, noise_idx, noise_start,
 *     snr_db: device arrays.  max_rir_len (host) sizes the partition count.  Limits, checked before any launch
 *     (DSK_ERR_INVALID): B >= 1, 1 <= L <= 2^24, 0 <= M <= DSK_AUG_MAX_SOURCES, 1 <= max_rir_len <= DSK_AUG_MAX_RIR,
 *     non-null pointers (the RIR bank only with rir_idx, the noise arrays only with M > 0).  No host synchronisation,
 *     no pageable copy; scratch is stream-ordered (cudaMallocAsync / cudaFreeAsync).
 *   dsk_fbank_segments: out (B, 1, T, 64) fp32, T = dsk_fbank_num_frames(L, sample_rate), the features of the B
 *     segments audio (B, L) fp32: row b is dsk_fbank on audio[b] alone (pre-emphasis from the segment's first sample;
 *     with subtract_mean, the mean over the segment's own T frames), then the SpecAugment masks exactly as
 *     dsk_fbank_crops applies them.  fb: the device copy of dsk_fbank_filterbank(sample_rate).  No host
 *     synchronisation.  For training, take L = flen + (T - 1) step samples (25 840 at 16 kHz for T = 160). */
#define DSK_AUG_MAX_SOURCES 8
#define DSK_AUG_MAX_RIR 65536
int32_t dsk_fbank_filterbank(int32_t sample_rate, float* fb);
int32_t dsk_wave_augment(const int16_t* speech, const int64_t* speech_off, int32_t U, const int64_t* utt,
                         const int64_t* start, int32_t B, int32_t L, const float* rir, const int64_t* rir_off, int32_t R,
                         int32_t max_rir_len, const int64_t* rir_idx, const int16_t* noise, const int64_t* noise_off,
                         int32_t N, int32_t M, const int64_t* noise_idx, const int64_t* noise_start, const double* snr_db,
                         float* out, void* stream);
int32_t dsk_fbank_segments(const float* audio, int32_t B, int32_t L, int32_t sample_rate, int32_t log_scale,
                           int32_t subtract_mean, const float* fb, const int32_t* time_masks, int32_t n_time,
                           const int32_t* freq_masks, int32_t n_freq, float* out, void* stream);

/* Threshold sweep of the verification metric (reference eval_metrics.py:16-37 calculate_roc, :53-88 calculate_val /
 * calculate_val_far; called from train_triplet.py:361): for every threshold t (double, as numpy's arange yields them)
 * tp[t] = #{i : same[i] && (double)dist[i] < t}, fp[t] = #{i : !same[i] && (double)dist[i] < t} — numpy's
 * np.less(dist, t) with its float32 -> float64 promotion, so the counts are exactly the reference's.  All other sweep
 * quantities (tn, fn, tpr, fpr, accuracy, val, far) are integer arithmetic on tp, fp, n_same, n_diff. */
int32_t dsk_threshold_counts(const float* dist, const uint8_t* same, int32_t P, const double* thresholds, int32_t nT,
                             int32_t* tp, int32_t* fp, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DSK_H_ */
