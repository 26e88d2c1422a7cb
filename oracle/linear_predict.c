/*
 * Oracle (test infrastructure only): plain-C restatement of scikit-learn's linear-classifier predict,
 *     scores = X @ coef_.T + intercept_ ; idx = argmax(scores, axis=1)          (first maximum wins, like np.argmax)
 * following sklearn/linear_model/_base.py:366-427 (the arithmetic behind the reference's canonical predictor,
 * unionml:README.md:87-92).  float64 throughout, one sequential FMA-free dot product per (row, class) in
 * feature order - the summation order differs from OpenBLAS' blocked dgemm, which only matters for gaps below ~1e-13
 * (tests/test_oracle_golden.py pins it against numpy and scikit-learn on seeded batches).
 *
 * Used by tests and by bench.py's cpu_baseline leg as a multi-threaded "what the host cores can do" number; never
 * linked into the product.  Build: gcc -O3 -fopenmp -shared -fPIC (recipe in __graft_entry__.build()).
 */
#include <stdint.h>

#ifdef _OPENMP
#include <omp.h>
#endif

/* binary models (n_classes == 1) use the `scores > 0` rule of _base.py:416 */
void oracle_linear_predict_f64(const double* x, int64_t n_rows, int n_features, const double* coef,
                               const double* intercept, int n_classes, int32_t* out) {
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < n_rows; ++r) {
    const double* xr = x + r * (int64_t)n_features;
    if (n_classes == 1) {
      double s = 0.0;
      for (int f = 0; f < n_features; ++f) s += xr[f] * coef[f];
      s += intercept[0];
      out[r] = s > 0.0 ? 1 : 0;
      continue;
    }
    int best = 0;
    double best_s = 0.0;
    for (int c = 0; c < n_classes; ++c) {
      const double* w = coef + (int64_t)c * n_features;
      double s = 0.0;
      for (int f = 0; f < n_features; ++f) s += xr[f] * w[f];
      s += intercept[c];
      if (c == 0 || s > best_s) {
        best = c;
        best_s = s;
      }
    }
    out[r] = best;
  }
}

/* same with float32 rows (the resident layout of the engine), promoted to float64 like numpy does for f32 @ f64 */
void oracle_linear_predict_f32(const float* x, int64_t n_rows, int n_features, const double* coef,
                               const double* intercept, int n_classes, int32_t* out) {
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < n_rows; ++r) {
    const float* xr = x + r * (int64_t)n_features;
    int best = 0;
    double best_s = 0.0;
    for (int c = 0; c < (n_classes == 1 ? 1 : n_classes); ++c) {
      const double* w = coef + (int64_t)c * n_features;
      double s = 0.0;
      for (int f = 0; f < n_features; ++f) s += (double)xr[f] * w[f];
      s += intercept[c];
      if (c == 0 || s > best_s) {
        best = c;
        best_s = s;
      }
    }
    out[r] = n_classes == 1 ? (best_s > 0.0 ? 1 : 0) : best;
  }
}

int oracle_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
