// Distance / triplet-loss / selection kernels (fp32).
// The summation orders are part of the contract: oracle/dsk_oracle.c restates them step by step so
// that the selection indices are bit-exact between GPU and oracle.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dsk_ptx.cuh"

namespace dsk {

// Canonical row reduction used by every distance in this file:
//   lane l accumulates fmaf(d,d,acc) over j = l, l+32, l+64, ... ; then xor-butterfly 16,8,4,2,1.
__device__ __forceinline__ float row_sqdist(const float* __restrict__ a, const float* __restrict__ b, int D,
                                            int lane) {
  float acc = 0.f;
  for (int j = lane; j < D; j += 32) {
    const float d = a[j] - b[j];
    acc = fmaf(d, d, acc);
  }
  for (int o = 16; o > 0; o >>= 1) acc = acc + __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

// PairwiseDistance(2).forward, reference model.py:13-18.  One warp per row.
__global__ void pairwise_distance_kernel(const float* __restrict__ x1, const float* __restrict__ x2, int B, int D,
                                         float eps, float* __restrict__ out) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B) return;
  const int lane = threadIdx.x & 31;
  const float s = row_sqdist(x1 + static_cast<long>(row) * D, x2 + static_cast<long>(row) * D, D, lane);
  if (lane == 0) out[row] = sqrtf(s + eps);
}

// grad_x1 = grad_out * (x1-x2)/dist ; grad_x2 = -grad_x1.
__global__ void pairwise_distance_bwd_kernel(const float* __restrict__ x1, const float* __restrict__ x2,
                                             const float* __restrict__ dist, const float* __restrict__ go, int B,
                                             int D, float* __restrict__ g1, float* __restrict__ g2) {
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long>(B) * D) return;
  const int row = i / D;
  const float g = go[row] * (x1[i] - x2[i]) / dist[row];
  if (g1) g1[i] = g;
  if (g2) g2[i] = -g;
}

// TripletMarginLoss.forward, reference model.py:27-33: d_p, d_n per row (one warp per row).
__global__ void triplet_dist_kernel(const float* __restrict__ a, const float* __restrict__ p,
                                    const float* __restrict__ n, int B, int D, float eps, float* __restrict__ d_p,
                                    float* __restrict__ d_n) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B) return;
  const int lane = threadIdx.x & 31;
  const long off = static_cast<long>(row) * D;
  const float sp = row_sqdist(a + off, p + off, D, lane);
  const float sn = row_sqdist(a + off, n + off, D, lane);
  if (lane == 0) {
    d_p[row] = sqrtf(sp + eps);
    d_n[row] = sqrtf(sn + eps);
  }
}

// loss = mean_i clamp(margin + d_p - d_n, min=0).  Single block, fixed reduction order.
__global__ void hinge_mean_kernel(const float* __restrict__ d_p, const float* __restrict__ d_n, int B, float margin,
                                  float* __restrict__ loss) {
  __shared__ float red[1024];
  float s = 0.f;
  for (int i = threadIdx.x; i < B; i += blockDim.x) s += fmaxf((margin + d_p[i]) - d_n[i], 0.f);
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = blockDim.x >> 1; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] = red[0] / static_cast<float>(B);
}

// d loss / d{a,p,n}.  torch.clamp(min=0) passes the gradient where its input >= 0.
__global__ void triplet_loss_bwd_kernel(const float* __restrict__ a, const float* __restrict__ p,
                                        const float* __restrict__ n, const float* __restrict__ d_p,
                                        const float* __restrict__ d_n, const float* __restrict__ grad_loss, int B,
                                        int D, float margin, float* __restrict__ ga, float* __restrict__ gp,
                                        float* __restrict__ gn) {
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long>(B) * D) return;
  const int row = i / D;
  const float dp = d_p[row], dn = d_n[row];
  const float active = ((margin + dp) - dn >= 0.f) ? 1.f : 0.f;
  const float g = active * grad_loss[0] / static_cast<float>(B);
  const float up = g * (a[i] - p[i]) / dp;   // d loss / d a via d_p
  const float un = -g * (a[i] - n[i]) / dn;  // d loss / d a via -d_n
  ga[i] = up + un;
  gp[i] = -up;
  gn[i] = -un;
}

// idx = ascending { i : d_n[i] - d_p[i] < margin }  == np.where(mask == 1), train_triplet.py:251-262.
// Single block; ordered compaction with warp ballots + a block scan per 1024-element chunk.
__global__ void margin_select_kernel(const float* __restrict__ d_p, const float* __restrict__ d_n, int B,
                                     float margin, int64_t* __restrict__ idx, int32_t* __restrict__ count) {
  __shared__ int warp_cnt[32];
  __shared__ int base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int start = 0; start < B; start += blockDim.x) {
    const int i = start + threadIdx.x;
    const bool sel = (i < B) && ((d_n[i] - d_p[i]) < margin);
    const unsigned m = __ballot_sync(0xffffffffu, sel);
    if (lane == 0) warp_cnt[warp] = __popc(m);
    __syncthreads();
    int off = base;
    for (int w = 0; w < warp; ++w) off += warp_cnt[w];
    if (sel) idx[off + __popc(m & ((1u << lane) - 1u))] = i;
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
      for (int w = 0; w < nwarps; ++w) t += warp_cnt[w];
      base += t;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) count[0] = base;
}

__global__ void gather_rows_kernel(const float* __restrict__ src, const int64_t* __restrict__ idx,
                                   const int32_t* __restrict__ count, int64_t row_elems, float* __restrict__ out) {
  const int j = blockIdx.x;
  if (j >= count[0]) return;
  const float* s = src + idx[j] * row_elems;
  float* o = out + static_cast<int64_t>(j) * row_elems;
  for (int64_t e = threadIdx.x; e < row_elems; e += blockDim.x) o[e] = s[e];
}

// ---------------------------------------------------------------------------------------------
// All-pairs distances (fp32, direct differences, sequential-in-d fmaf order) of the anchor rows [row0, row0 + rows)
// against all N rows into a dense rows x N matrix, 64x64 tile per block of 256 threads (4x4 outputs per thread).
// Every element depends only on its two rows, so any row range gives the bits of the full N x N matrix.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
allpairs_sqdist_kernel(const float* __restrict__ E, int N, int D, int row0, int rows, float* __restrict__ S) {
  constexpr int TM = 64, TK = 16;
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TM + 4];
  const int i0 = row0 + blockIdx.y * TM, j0 = blockIdx.x * TM, row_end = row0 + rows;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
  for (int k0 = 0; k0 < D; k0 += TK) {
    for (int t = threadIdx.x; t < TM * TK; t += 256) {
      const int r = t / TK, k = t % TK;
      As[k][r] = (i0 + r < row_end && k0 + k < D) ? E[static_cast<long>(i0 + r) * D + k0 + k] : 0.f;
      Bs[k][r] = (j0 + r < N && k0 + k < D) ? E[static_cast<long>(j0 + r) * D + k0 + k] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      float av[4], bv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) av[r] = As[k][ty * 4 + r];
#pragma unroll
      for (int c = 0; c < 4; ++c) bv[c] = Bs[k][tx * 4 + c];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float d = av[r] - bv[c];
          acc[r][c] = fmaf(d, d, acc[r][c]);
        }
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int i = i0 + ty * 4 + r, j = j0 + tx * 4 + c;
      if (i < row_end && j < N) S[static_cast<long>(i - row0) * N + j] = acc[r][c];
    }
}

// Per anchor row0 + i (i < rows): the k smallest sqrt(S+eps) among columns with a different label, ties -> lower
// column.  S is the rows x N matrix of allpairs_sqdist_kernel; idx / val are written at local row i.
// One warp per row; each pass extracts the lexicographic (value, index) minimum.
__global__ void topk_rows_kernel(const float* __restrict__ S, const int64_t* __restrict__ labels, int N, int row0,
                                 int rows, float eps, int k, int64_t* __restrict__ idx, float* __restrict__ val) {
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= rows) return;
  const int row = row0 + i;
  const int lane = threadIdx.x & 31;
  const float* s = S + static_cast<long>(i) * N;
  const int64_t my_label = labels[row];
  float last_v = -1.f;
  int last_j = -1;
  for (int t = 0; t < k; ++t) {
    float bv = __int_as_float(0x7f800000);  // +inf
    int bj = 0x7fffffff;
    for (int j = lane; j < N; j += 32) {
      if (labels[j] == my_label) continue;
      const float v = sqrtf(s[j] + eps);
      // strictly after (last_v, last_j) in lexicographic order
      const bool after = (v > last_v) || (v == last_v && j > last_j);
      if (after && (v < bv || (v == bv && j < bj))) {
        bv = v;
        bj = j;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (ov < bv || (ov == bv && oj < bj)) {
        bv = ov;
        bj = oj;
      }
    }
    if (lane == 0) {
      idx[static_cast<long>(i) * k + t] = (bj == 0x7fffffff) ? -1 : bj;
      val[static_cast<long>(i) * k + t] = bv;
    }
    last_v = bv;
    last_j = bj;
  }
}

}  // namespace dsk

// =================================================================================================
// Tensor-core all-pairs path: fp16 Gram on wgmma (conv_umma_kernel used as a plain GEMM, fp32 output), candidate
// selection from the approximate distances, EXACT fp32 refinement of the candidates in the canonical order of
// allpairs_sqdist_kernel (sequential-in-d fmaf), so the result is bit-identical to the exact path / the oracle.
// =================================================================================================
namespace dsk {

// E fp32 [N][D] -> 16-bit [Npad][D] (rows >= N zero) + squared norms of the ROUNDED rows. One block per row.
template <bool BF16>
__global__ void allpairs_prep_kernel(const float* __restrict__ E, int N, int D, uint16_t* __restrict__ E16,
                                     float* __restrict__ norms) {
  __shared__ float red[32];
  const int row = blockIdx.x;
  float s = 0.f;
  for (int t = threadIdx.x; t < D; t += blockDim.x) {
    uint16_t h = 0;
    if (row < N) {
      h = to16<BF16>(E[static_cast<long>(row) * D + t]);
      const float f = from16<BF16>(h);
      s = fmaf(f, f, s);
    }
    E16[static_cast<long>(row) * D + t] = h;
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) t += red[w];
    norms[row] = t;
  }
}

constexpr int kApCand = 16;  // candidates refined exactly per row (must be >= k; host enforces k <= 8)

__device__ __forceinline__ float exact_dist_seq(const float* __restrict__ a, const float* __restrict__ b, int D,
                                                float eps) {
  float acc = 0.f;
  for (int t = 0; t < D; ++t) {
    const float d = a[t] - b[t];
    acc = fmaf(d, d, acc);
  }
  return sqrtf(acc + eps);
}

// One warp per anchor row0 + i (i < rows).  G: fp32 Gram of the rounded anchor rows against all rounded rows
// [rows_pad][Npad] (local row i); approximate squared distance
// a_ij = n_i + n_j - 2 G_ij (exact squared distance of the ROUNDED rows up to fp32 accumulation).
// Exactness argument: rounding row e to 16 bit moves it by at most u*||e|| (u = unit roundoff), so for every pair
//   | a_ij - ||e_i - e_j||^2 | <= 2 d r + r^2 + slack,   r = u (||e_i|| + max_j ||e_j||),  d = ||e_i - e_j||.
// If the worst kept candidate's a exceeds (k-th exact distance)^2 by more than that bound, no discarded column can
// beat the k-th result and the refined top-k is the exact answer; otherwise the warp scans the whole row exactly.  A row
// with fewer valid columns than kApCand refines them all.  The bound says nothing once a norm or an approximate distance
// is not finite (an fp16 entry of magnitude >= 65520 rounds to inf while the fp32 distance is finite): such a row scans.
// Either way the result is the exact one, whatever the Gram's bits: idx / val (written at local row i) do not depend on
// the row range the Gram was computed for.  ROWS = false is the whole batch (row0 = 0, rows = N, the arguments are
// ignored): dsk_allpairs_topk_tc and the whole-batch loss run the instruction stream they ran before the row range
// existed, without the offset arithmetic in this latency-bound kernel.
template <bool ROWS>
__global__ void __launch_bounds__(256)
allpairs_select_refine_kernel(const float* __restrict__ E, const float* __restrict__ G, const float* __restrict__ norms,
                              const int64_t* __restrict__ labels, int N, int Npad, int row0_arg, int rows_arg, int D,
                              float eps, int k, float u, int64_t* __restrict__ idx, float* __restrict__ val) {
  __shared__ int cand_j[8][kApCand];
  __shared__ float cand_a[8][kApCand];
  const int row0 = ROWS ? row0_arg : 0, rows = ROWS ? rows_arg : N;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + w;
  if (i >= rows) return;
  const int row = row0 + i;
  const float* g = G + static_cast<long>(i) * Npad;
  const float ni = norms[row];
  const int64_t my_label = labels[row];
  const float INF = __int_as_float(0x7f800000);
  // Valid (other-label) columns of the row, and whether any has a non-finite approximate distance (a 16-bit overflow
  // of an entry makes a norm inf; such a column is never a candidate, so the row must take the exact scan).
  int n_valid = 0;
  bool nonfinite = false;
  // ---- candidates: the kApCand smallest approximate distances, extracted in lexicographic (a, j) order.
  // Rows of up to 1024 columns keep their 32 values per lane in registers; longer rows re-read G (L1/L2 hits).
  constexpr int kRegCols = 32;
  const bool in_regs = N <= 32 * kRegCols;
  float areg[kRegCols];
  if (in_regs) {
#pragma unroll
    for (int q = 0; q < kRegCols; ++q) {
      const int j = lane + 32 * q;
      const bool valid = j < N && labels[j] != my_label;
      const float a = valid ? (ni + norms[j]) - 2.0f * g[j] : INF;
      n_valid += valid;
      nonfinite |= valid && !(fabsf(a) < INF);
      areg[q] = a;
    }
  } else {
    for (int j = lane; j < N; j += 32) {
      if (labels[j] == my_label) continue;
      ++n_valid;
      nonfinite |= !(fabsf((ni + norms[j]) - 2.0f * g[j]) < INF);
    }
  }
  n_valid = __reduce_add_sync(0xffffffffu, n_valid);
  nonfinite = __any_sync(0xffffffffu, nonfinite);
  float last_a = -INF;
  int last_j = -1;
  for (int t = 0; t < kApCand; ++t) {
    float ba = INF;
    int bj = 0x7fffffff;
    if (in_regs) {
#pragma unroll
      for (int q = 0; q < kRegCols; ++q) {
        const int j = lane + 32 * q;
        const float a = areg[q];
        const bool after = (a > last_a) || (a == last_a && j > last_j);
        if (a < INF && after && (a < ba || (a == ba && j < bj))) {
          ba = a;
          bj = j;
        }
      }
    } else {
      for (int j = lane; j < N; j += 32) {
        if (labels[j] == my_label) continue;
        const float a = (ni + norms[j]) - 2.0f * g[j];
        const bool after = (a > last_a) || (a == last_a && j > last_j);
        if (after && (a < ba || (a == ba && j < bj))) {
          ba = a;
          bj = j;
        }
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float oa = __shfl_xor_sync(0xffffffffu, ba, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (oa < ba || (oa == ba && oj < bj)) {
        ba = oa;
        bj = oj;
      }
    }
    if (lane == 0) {
      cand_j[w][t] = bj;
      cand_a[w][t] = ba;
    }
    last_a = ba;
    last_j = bj;
  }
  __syncwarp();
  // ---- exact refinement of the candidates (lane t < kApCand owns candidate t)
  float v = INF;
  int j = 0x7fffffff;
  if (lane < kApCand && cand_j[w][lane] != 0x7fffffff) {
    j = cand_j[w][lane];
    v = exact_dist_seq(E + static_cast<long>(row) * D, E + static_cast<long>(j) * D, D, eps);
  }
  // k-th smallest exact value among the candidates
  float kth = INF;
  {
    float lv = -1.f;
    int lj = -1;
    for (int t = 0; t < k; ++t) {
      float bv = INF;
      int bj = 0x7fffffff;
      const bool after = (v > lv) || (v == lv && j > lj);
      if (after) {
        bv = v;
        bj = j;
      }
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
        if (ov < bv || (ov == bv && oj < bj)) {
          bv = ov;
          bj = oj;
        }
      }
      lv = bv;
      lj = bj;
      kth = bv;
    }
  }
  // safe iff every column NOT among the candidates has approximate squared distance >= kth^2 + bound
  const float worst_a = cand_a[w][kApCand - 1];
  float nmax = 0.f;
  for (int jj = lane; jj < N; jj += 32) nmax = fmaxf(nmax, norms[jj]);
  for (int o = 16; o > 0; o >>= 1) nmax = fmaxf(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
  const float r = u * (sqrtf(ni) + sqrtf(nmax)) * 1.01f;
  const float dmax = sqrtf(fmaxf(worst_a, 0.f)) + r + 1e-3f;
  const float tol = 2.f * dmax * r + r * r + 1e-5f * (ni + nmax) + 1e-4f;
  // the candidates are every valid column, or no discarded one can come closer than the k-th; non-finite norms or
  // approximate distances void both arguments
  const bool finite = !nonfinite && fabsf(ni) < INF && fabsf(nmax) < INF;
  const bool all_candidates = n_valid < kApCand;
  const bool safe = finite && (all_candidates || worst_a >= (kth * kth - eps) + tol);
  if (!safe) {
    // ---- exact fallback: scan the whole row (rare); same arithmetic as the exact path
    float lv = -1.f;
    int lj = -1;
    for (int t = 0; t < k; ++t) {
      float bv = INF;
      int bj = 0x7fffffff;
      for (int jj = lane; jj < N; jj += 32) {
        if (labels[jj] == my_label) continue;
        const float vv = exact_dist_seq(E + static_cast<long>(row) * D, E + static_cast<long>(jj) * D, D, eps);
        const bool after = (vv > lv) || (vv == lv && jj > lj);
        if (after && (vv < bv || (vv == bv && jj < bj))) {
          bv = vv;
          bj = jj;
        }
      }
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
        if (ov < bv || (ov == bv && oj < bj)) {
          bv = ov;
          bj = oj;
        }
      }
      if (lane == 0) {
        idx[static_cast<long>(i) * k + t] = (bj == 0x7fffffff) ? -1 : bj;
        val[static_cast<long>(i) * k + t] = bv;
      }
      lv = bv;
      lj = bj;
    }
    return;
  }
  // ---- final top-k among the exactly refined candidates, (value, index) lexicographic
  float lv = -1.f;
  int lj = -1;
  for (int t = 0; t < k; ++t) {
    float bv = INF;
    int bj = 0x7fffffff;
    const bool after = (v > lv) || (v == lv && j > lj);
    if (after) {
      bv = v;
      bj = j;
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (ov < bv || (ov == bv && oj < bj)) {
        bv = ov;
        bj = oj;
      }
    }
    if (lane == 0) {
      idx[static_cast<long>(i) * k + t] = (bj == 0x7fffffff) ? -1 : bj;
      val[static_cast<long>(i) * k + t] = bv;
    }
    lv = bv;
    lj = bj;
  }
}

// =================================================================================================
// Batch-hard triplet loss over one batch of N embeddings: every anchor i takes its hardest positive (farthest same-label
// row) and its hardest negative (nearest different-label row) inside the batch.  Distances are those of the all-pairs
// ops above, bit for bit.  The negative is the k = 1 result of allpairs_select_refine_kernel / topk_rows_kernel.
// =================================================================================================

// Hardest positive, one warp per anchor: argmax over j != i with labels[j] == labels[i] of the exact distance, ties ->
// lower j (FROM_S: sqrt(S[i][j] + eps) from allpairs_sqdist_kernel, else exact_dist_seq; the two are the same bits).
// pos_idx = -1 and d_ap = 0 when the anchor has no positive.  valid[i] = 1 iff it has a positive and a negative.
// Anchors row0 + i for i < rows; S (rows x N) and the outputs are indexed by the local row i, column indices are global.
template <bool FROM_S>
__global__ void __launch_bounds__(256)
batch_hard_positive_kernel(const float* __restrict__ E, const float* __restrict__ S, const int64_t* __restrict__ labels,
                           int N, int row0, int rows, int D, float eps, int64_t* __restrict__ pos_idx,
                           float* __restrict__ d_ap, uint8_t* __restrict__ valid) {
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= rows) return;
  const int row = row0 + i;
  const int lane = threadIdx.x & 31;
  const int64_t my_label = labels[row];
  float bv = -1.f;  // below every distance (>= sqrt(eps) > 0)
  int bj = 0x7fffffff;
  bool has_neg = false;
  for (int j = lane; j < N; j += 32) {
    if (labels[j] != my_label) {
      has_neg = true;
      continue;
    }
    if (j == row) continue;
    const float v = FROM_S ? sqrtf(S[static_cast<long>(i) * N + j] + eps)
                           : exact_dist_seq(E + static_cast<long>(row) * D, E + static_cast<long>(j) * D, D, eps);
    if (v > bv) {  // each lane scans ascending j: strict > keeps the lower index of a tie
      bv = v;
      bj = j;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
    if (ov > bv || (ov == bv && oj < bj)) {
      bv = ov;
      bj = oj;
    }
  }
  has_neg = __any_sync(0xffffffffu, has_neg);
  if (lane == 0) {
    const bool has_pos = bj != 0x7fffffff;
    pos_idx[i] = has_pos ? bj : -1;
    d_ap[i] = has_pos ? bv : 0.f;
    valid[i] = (has_pos && has_neg) ? 1 : 0;
  }
}

// loss = (1/V) sum over valid anchors of clamp(margin + d_ap - d_an, 0), V = number of valid anchors (loss 0 when
// V = 0).  Single block of 1024 threads, the order of hinge_mean_kernel: strided partial sums, then a halving tree.
__global__ void __launch_bounds__(1024)
batch_hard_mean_kernel(const float* __restrict__ d_ap, const float* __restrict__ d_an,
                       const uint8_t* __restrict__ valid, int N, float margin, float* __restrict__ loss) {
  __shared__ float red[1024];
  __shared__ int cnt[1024];
  float s = 0.f;
  int c = 0;
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    if (valid[i]) {
      s += fmaxf((margin + d_ap[i]) - d_an[i], 0.f);
      ++c;
    }
  red[threadIdx.x] = s;
  cnt[threadIdx.x] = c;
  __syncthreads();
  for (int o = blockDim.x >> 1; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      red[threadIdx.x] += red[threadIdx.x + o];
      cnt[threadIdx.x] += cnt[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] = cnt[0] > 0 ? red[0] / static_cast<float>(cnt[0]) : 0.f;
}

// coef[0] = grad_loss / V (0 when V = 0): the weight of every anchor whose hinge passes the gradient.  Single block.
__global__ void __launch_bounds__(1024)
batch_hard_coef_kernel(const uint8_t* __restrict__ valid, int N, const float* __restrict__ grad_loss,
                       float* __restrict__ coef) {
  __shared__ int cnt[1024];
  int c = 0;
  for (int i = threadIdx.x; i < N; i += blockDim.x) c += valid[i] ? 1 : 0;
  cnt[threadIdx.x] = c;
  __syncthreads();
  for (int o = blockDim.x >> 1; o > 0; o >>= 1) {
    if (threadIdx.x < o) cnt[threadIdx.x] += cnt[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) coef[0] = cnt[0] > 0 ? grad_loss[0] / static_cast<float>(cnt[0]) : 0.f;
}

// The hinge passes the gradient where margin + d_ap - d_an >= 0 (torch.clamp(min=0), as triplet_loss_bwd_kernel).
__device__ __forceinline__ bool batch_hard_active(const uint8_t* valid, const float* d_ap, const float* d_an, int i,
                                                  float margin) {
  return valid[i] && ((margin + d_ap[i]) - d_an[i] >= 0.f);
}

// gE[j] (written, not accumulated), one block of 128 threads per row j, thread t owning elements t, t+128, ...
// Fixed order per row, no float atomics: row j's own anchor term first, then the terms of the anchors that chose j as
// their positive or negative in ascending anchor order.  That inverse list is built on the device chunk by chunk: each
// chunk of 128 anchors is compacted (warp ballots + a block prefix, stable) into shared memory, then applied.  A row that
// many anchors chose (a hub) only makes its own block longer.  Terms, with g = coef[0] and one division per term:
//   anchor a:  (g / d_ap) (a - p) - (g / d_an) (a - n);   its positive p: -(g / d_ap) (a - p);   its negative n: +(g / d_an) (a - n).
// The chooser's thread divides while the list is built, so the apply loop holds no division call (no spill).
// Block b computes row j = row0 + b into gE[b]; the selection arrays cover all N anchors, so any row range gives the
// bits of the full gradient.
__global__ void __launch_bounds__(128)
batch_hard_bwd_kernel(const float* __restrict__ E, const int64_t* __restrict__ pos_idx,
                      const int64_t* __restrict__ neg_idx, const float* __restrict__ d_ap,
                      const float* __restrict__ d_an, const uint8_t* __restrict__ valid, int N, int D, int row0,
                      float margin, const float* __restrict__ coef, float* __restrict__ gE) {
  __shared__ int list[128];     // anchors that chose row j, ascending
  __shared__ float scale[128];  // their signed coefficients: -(g / d_ap) if j is the positive, +(g / d_an) if the negative
  __shared__ int wcnt[4];
  const int j = row0 + blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float g = coef[0];
  const float* ej = E + static_cast<long>(j) * D;
  float* gj = gE + static_cast<long>(blockIdx.x) * D;
  if (batch_hard_active(valid, d_ap, d_an, j, margin)) {
    const float* ep = E + pos_idx[j] * D;
    const float* en = E + neg_idx[j] * D;
    const float sp = g / d_ap[j], sn = g / d_an[j];
    for (int d = threadIdx.x; d < D; d += 128) gj[d] = sp * (ej[d] - ep[d]) - sn * (ej[d] - en[d]);
  } else {
    for (int d = threadIdx.x; d < D; d += 128) gj[d] = 0.f;
  }
  for (int base = 0; base < N; base += 128) {
    const int i = base + threadIdx.x;
    bool chose = false;
    float sc = 0.f;
    if (i < N && batch_hard_active(valid, d_ap, d_an, i, margin)) {
      if (pos_idx[i] == j) {
        chose = true;
        sc = -(g / d_ap[i]);
      } else if (neg_idx[i] == j) {
        chose = true;
        sc = g / d_an[i];
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, chose);
    if (lane == 0) wcnt[warp] = __popc(m);
    __syncthreads();
    int off = 0, total = 0;
    for (int w = 0; w < 4; ++w) {
      off += w < warp ? wcnt[w] : 0;
      total += wcnt[w];
    }
    if (chose) {
      const int at = off + __popc(m & ((1u << lane) - 1u));
      list[at] = i;
      scale[at] = sc;
    }
    __syncthreads();
    for (int e = 0; e < total; ++e) {
      const float* ea = E + static_cast<long>(list[e]) * D;
      const float sc = scale[e];
      for (int d = threadIdx.x; d < D; d += 128) gj[d] += sc * (ea[d] - ej[d]);
    }
    __syncthreads();  // list, scale and wcnt are rewritten by the next chunk
  }
}

}  // namespace dsk
