/*
 * Oracle SpMM (TEST INFRASTRUCTURE, see oracle/__init__.py).
 *
 * CPU restatement of DGL's `update_all(fn.copy_src, fn.sum)` as used at
 * PipeGCN/module/layer.py:47-49 (and its backward on the reversed graph):
 *     out[r, :] = sum over e in [indptr[r], indptr[r+1]) of x[indices[e], :]
 * DGL is absent from PipeGCN (fork chwan-rice/dgl, unpinned); copy_src + sum
 * over a 0/1 adjacency is exactly this row-wise sum.  fp32 accumulation in edge order,
 * rows distributed over OpenMP threads (DGL's CPU SpMM is OpenMP-parallel over rows too).
 */
#include <omp.h>
#include <stdint.h>
#include <string.h>

/* torchrun exports OMP_NUM_THREADS=1 to its workers: the CPU baseline sets its thread count explicitly */
void oracle_set_threads(int n) { if (n > 0) omp_set_num_threads(n); }
int oracle_get_max_threads(void) { return omp_get_max_threads(); }

void oracle_spmm_sum_f32(const int64_t* indptr, const int64_t* indices, const float* x, float* out,
                         int64_t n_rows, int64_t d) {
#pragma omp parallel for schedule(dynamic, 64)
  for (int64_t r = 0; r < n_rows; ++r) {
    float* o = out + r * d;
    memset(o, 0, sizeof(float) * (size_t)d);
    for (int64_t e = indptr[r]; e < indptr[r + 1]; ++e) {
      const float* s = x + indices[e] * d;
      for (int64_t k = 0; k < d; ++k) o[k] += s[k];
    }
  }
}
