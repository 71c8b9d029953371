/* oracle/ref_stub -- TEST INFRASTRUCTURE.  The part of cblas.h that caffe/util/
 * math_functions.hpp and mkl_alternate.hpp name: the enums, and element-wise host stand-ins for
 * the level-1 calls mkl_alternate.hpp wraps (x[i] * a, y[i] + a * x[i], one element at a time). */
#ifndef MNC_REF_STUB_CBLAS_H_
#define MNC_REF_STUB_CBLAS_H_
enum CBLAS_ORDER { CblasRowMajor = 101, CblasColMajor = 102 };
enum CBLAS_TRANSPOSE { CblasNoTrans = 111, CblasTrans = 112, CblasConjTrans = 113 };
inline void cblas_sscal(const int n, const float a, float* x, const int inc) {
  for (int i = 0; i < n; ++i) x[i * inc] *= a;
}
inline void cblas_dscal(const int n, const double a, double* x, const int inc) {
  for (int i = 0; i < n; ++i) x[i * inc] *= a;
}
inline void cblas_saxpy(const int n, const float a, const float* x, const int ix, float* y,
                        const int iy) {
  for (int i = 0; i < n; ++i) y[i * iy] += a * x[i * ix];
}
inline void cblas_daxpy(const int n, const double a, const double* x, const int ix, double* y,
                        const int iy) {
  for (int i = 0; i < n; ++i) y[i * iy] += a * x[i * ix];
}
#endif
