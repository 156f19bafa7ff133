/*
 * dsk_oracle.c — CPU restatement of the distance / triplet-loss / selection arithmetic.
 * TEST INFRASTRUCTURE ONLY: linked by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg,
 * never by the product library.
 *
 * Follows the reference formulas
 *   PairwiseDistance.forward     reference model.py:13-18   d = sqrt(sum |x1-x2|^2 + 1e-4/D)
 *   TripletMarginLoss.forward    reference model.py:27-33   mean(clamp(margin + d_p - d_n, 0))
 *   hard-triplet mask            reference train_triplet.py:251-262   where(d_n - d_p < margin)
 * and, for the all-pairs top-k of BASELINE config 4 (absent from the reference, parity unpinned),
 * the same PairwiseDistance formula over every pair.
 *
 * fp32 addition is not associative and the reference leaves the summation order to PyTorch, so this
 * file fixes one order and the CUDA kernels (csrc/loss_kernels.cuh) use exactly the same one:
 * that makes d_p, d_n and therefore the selected indices bit-identical between GPU and oracle.
 * The pinning against the reference's own outputs (tests/golden/triplet_loss.npz) is to 1e-6
 * relative on distances and exact on the index list.
 *
 * Build: gcc -O2 -ffp-contract=off -shared -fPIC -o _build/libdsk_oracle.so dsk_oracle.c -lm
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

/* lane l accumulates fmaf(d,d,acc) over j = l, l+32, ...; then xor-butterfly 16,8,4,2,1 (all lanes equal). */
static float row_sqdist(const float* a, const float* b, int D) {
  float part[32], tmp[32];
  for (int l = 0; l < 32; ++l) {
    float acc = 0.f;
    for (int j = l; j < D; j += 32) {
      const float d = a[j] - b[j];
      acc = fmaf(d, d, acc);
    }
    part[l] = acc;
  }
  for (int o = 16; o > 0; o >>= 1) {
    for (int l = 0; l < 32; ++l) tmp[l] = part[l] + part[l ^ o];
    for (int l = 0; l < 32; ++l) part[l] = tmp[l];
  }
  return part[0];
}

static float pd_eps(int D) { return (float)(1e-4 / (double)D); }

void orc_pairwise_distance(const float* x1, const float* x2, int B, int D, float* out) {
  const float eps = pd_eps(D);
  for (int i = 0; i < B; ++i) out[i] = sqrtf(row_sqdist(x1 + (long)i * D, x2 + (long)i * D, D) + eps);
}

/* loss: 1024 strided partial sums, then halving tree (the order of hinge_mean_kernel). */
void orc_triplet_loss(const float* a, const float* p, const float* n, int B, int D, float margin, float* loss,
                      float* d_p, float* d_n) {
  orc_pairwise_distance(a, p, B, D, d_p);
  orc_pairwise_distance(a, n, B, D, d_n);
  float red[1024];
  for (int t = 0; t < 1024; ++t) {
    float s = 0.f;
    for (int i = t; i < B; i += 1024) s += fmaxf((margin + d_p[i]) - d_n[i], 0.f);
    red[t] = s;
  }
  for (int o = 512; o > 0; o >>= 1)
    for (int t = 0; t < o; ++t) red[t] += red[t + o];
  loss[0] = red[0] / (float)B;
}

/* ascending indices with d_n - d_p < margin; returns the count. */
int orc_margin_select(const float* d_p, const float* d_n, int B, float margin, int64_t* idx) {
  int k = 0;
  for (int i = 0; i < B; ++i)
    if ((d_n[i] - d_p[i]) < margin) idx[k++] = i;
  return k;
}

/* all pairs, sequential-in-d fmaf accumulation; k smallest per row among different labels, ties -> lower j. */
void orc_allpairs_topk(const float* E, const int64_t* labels, int N, int D, int k, int64_t* idx, float* val) {
  const float eps = pd_eps(D);
  float* drow = (float*)malloc(sizeof(float) * (size_t)N);
  for (int i = 0; i < N; ++i) {
    const float* ei = E + (long)i * D;
    for (int j = 0; j < N; ++j) {
      const float* ej = E + (long)j * D;
      float acc = 0.f;
      for (int d = 0; d < D; ++d) {
        const float df = ei[d] - ej[d];
        acc = fmaf(df, df, acc);
      }
      drow[j] = sqrtf(acc + eps);
    }
    float last_v = -1.f;
    int last_j = -1;
    for (int t = 0; t < k; ++t) {
      float bv = INFINITY;
      int bj = -1;
      for (int j = 0; j < N; ++j) {
        if (labels[j] == labels[i]) continue;
        const float v = drow[j];
        const int after = (v > last_v) || (v == last_v && j > last_j);
        if (after && (bj < 0 || v < bv)) { /* ascending j scan: strict < keeps the lowest index on ties */
          bv = v;
          bj = j;
        }
      }
      idx[(long)i * k + t] = bj;
      val[(long)i * k + t] = bv;
      last_v = bv;
      last_j = bj;
    }
  }
  free(drow);
}
