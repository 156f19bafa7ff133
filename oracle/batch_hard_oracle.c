/*
 * batch_hard_oracle.c — CPU restatement of the batch-hard triplet loss (dsk_batch_hard_triplet).
 * TEST INFRASTRUCTURE ONLY: linked by tests/, never by the product library.
 *
 * The reference has no batch-hard loss (parity with it is unpinned).  The definition is built from
 * PairwiseDistance (reference model.py:13-18) and the hinge of TripletMarginLoss (model.py:27-33):
 *   d(i,j)   = sqrtf(sum_d fmaf-sequential (E_i - E_j)^2 + 1e-4/D)   (the all-pairs distance of dsk_oracle.c)
 *   pos_i    = argmax d(i,j) over j != i, label_j == label_i      ties -> lower j   (-1, d_ap = 0 if none)
 *   neg_i    = argmin d(i,j) over label_j != label_i              ties -> lower j   (-1, d_an = +inf if none)
 *              (a NaN distance is never selected)
 *   valid_i  = pos_i exists and some label_j != label_i
 *   a row i holding a NaN or an infinity: d_ap = d_an = NaN, valid_i = some j != i with label_j == label_i and some
 *              label_j != label_i, pos_i / neg_i as above
 *   loss     = (1/V) sum_{valid i} clamp(margin + d_ap - d_an, 0) (NaN stays NaN), V = #valid, 0 when V = 0,
 * summed in the order of batch_hard_mean_kernel (csrc/loss_kernels.cuh): 1024 strided partial sums in ascending i,
 * then a halving tree.
 *
 * Build: gcc -O2 -ffp-contract=off -shared -fPIC -o _build/libbatch_hard_oracle.so batch_hard_oracle.c -lm
 */
#include <math.h>
#include <stdint.h>

static float dist(const float* a, const float* b, int D, float eps) {
  float acc = 0.f;
  for (int d = 0; d < D; ++d) {
    const float df = a[d] - b[d];
    acc = fmaf(df, df, acc);
  }
  return sqrtf(acc + eps);
}

void orc_batch_hard_triplet(const float* E, const int64_t* labels, int N, int D, float margin, float* loss,
                            int64_t* pos_idx, int64_t* neg_idx, float* d_ap, float* d_an, uint8_t* valid) {
  const float eps = (float)(1e-4 / (double)D);
  for (int i = 0; i < N; ++i) {
    const float* ei = E + (long)i * D;
    int pj = -1, nj = -1, has_same = 0, has_neg = 0, nonfinite = 0;
    float pv = -1.f, nv = INFINITY;
    for (int d = 0; d < D; ++d) nonfinite |= !isfinite(ei[d]);
    for (int j = 0; j < N; ++j) { /* ascending j: strict comparisons keep the lower index of a tie */
      if (labels[j] == labels[i]) {
        if (j == i) continue;
        has_same = 1;
        const float v = dist(ei, E + (long)j * D, D, eps);
        if (v > pv) {
          pv = v;
          pj = j;
        }
      } else {
        has_neg = 1;
        const float v = dist(ei, E + (long)j * D, D, eps);
        if ((nj < 0 && !isnan(v)) || v < nv) {
          nv = v;
          nj = j;
        }
      }
    }
    pos_idx[i] = pj;
    neg_idx[i] = nj;
    d_ap[i] = nonfinite ? NAN : pj >= 0 ? pv : 0.f;
    d_an[i] = nonfinite ? NAN : nv;
    valid[i] = ((nonfinite ? has_same : pj >= 0) && has_neg) ? 1 : 0;
  }
  float red[1024];
  int cnt[1024];
  for (int t = 0; t < 1024; ++t) {
    float s = 0.f;
    int c = 0;
    for (int i = t; i < N; i += 1024)
      if (valid[i]) {
        const float h = (margin + d_ap[i]) - d_an[i];
        s += isnan(h) ? h : fmaxf(h, 0.f);
        ++c;
      }
    red[t] = s;
    cnt[t] = c;
  }
  for (int o = 512; o > 0; o >>= 1)
    for (int t = 0; t < o; ++t) {
      red[t] += red[t + o];
      cnt[t] += cnt[t + o];
    }
  loss[0] = cnt[0] > 0 ? red[0] / (float)cnt[0] : 0.f;
}
