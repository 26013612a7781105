// Dynamical matrices D(q) of a periodic crystal from its compact force constants (CHGNet.phonons).
//
//   D(q)[k a, k' b] = sum_{j : s2p[j] = k'} Phi[k, j, a, b] (1/m_kj) sum_{v in images(k, j)} e^{2 pi i q.v}
//                     / sqrt(m_k m_k'),
//
// phonopy's phase convention: v = r_j - r_k (basis offsets included) in primitive fractional coordinates, one v per
// minimum image, m_kj their number.  The phases are generated and contracted in registers: the [Q, n_prim, N_super]
// phase tensor never exists.  One thread per (q, unordered pair {k, k'}): it sums the blocks (k, k') and (k', k) in
// fp64, in a fixed order, and writes both 3x3 blocks of the Hermitian part (D + D^H)/2.  No atomics: the result is
// bitwise reproducible.
#include "common.cuh"

namespace chg {
namespace {

constexpr int DYN_THREADS = 128;  // q-points per block

// re / im [3][3] = sum_{j : s2p[j] = kp} Phi[k, j] (1/m) sum_images e^{2 pi i q.v}
__device__ __forceinline__ void phase_block(const double* __restrict__ fc, const int32_t* __restrict__ img_ptr,
                                            const double* __restrict__ img_vec, const int32_t* __restrict__ s2p,
                                            int n_super, int k, int kp, double q0, double q1, double q2,
                                            double (&re)[9], double (&im)[9]) {
#pragma unroll
  for (int i = 0; i < 9; ++i) re[i] = im[i] = 0.0;
  // every thread of a block has the same (k, kp): the branch and the loads below are uniform across the warp
  for (int j = 0; j < n_super; ++j) {
    if (__ldg(s2p + j) != kp) continue;
    const size_t pair = (size_t)k * n_super + j;
    const int b = __ldg(img_ptr + pair), e = __ldg(img_ptr + pair + 1);
    if (e == b) continue;
    double c = 0.0, s = 0.0;
    for (int t = b; t < e; ++t) {
      const double* v = img_vec + (size_t)t * 3;
      double sn, cs;
      sincospi(2.0 * fma(q0, __ldg(v), fma(q1, __ldg(v + 1), q2 * __ldg(v + 2))), &sn, &cs);
      c += cs;
      s += sn;
    }
    const double inv_m = 1.0 / (double)(e - b);
    c *= inv_m;
    s *= inv_m;
    const double* f = fc + pair * 9;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const double x = __ldg(f + i);
      re[i] = fma(x, c, re[i]);
      im[i] = fma(x, s, im[i]);
    }
  }
}

__global__ void __launch_bounds__(DYN_THREADS)
dynamical_matrices_kernel(const double* __restrict__ fc, const int32_t* __restrict__ img_ptr,
                          const double* __restrict__ img_vec, const int32_t* __restrict__ s2p,
                          const double* __restrict__ inv_sqrt_m, int n_prim, int n_super,
                          const double* __restrict__ qpoints, int n_q, double* __restrict__ dyn) {
  const int k = blockIdx.x / n_prim, kp = blockIdx.x % n_prim;
  if (kp < k) return;  // block (kp, k) writes this pair
  const int iq = blockIdx.y * DYN_THREADS + threadIdx.x;
  if (iq >= n_q) return;
  const double q0 = qpoints[iq * 3], q1 = qpoints[iq * 3 + 1], q2 = qpoints[iq * 3 + 2];
  double r1[9], i1[9], r2[9], i2[9];
  phase_block(fc, img_ptr, img_vec, s2p, n_super, k, kp, q0, q1, q2, r1, i1);
  if (kp != k) {
    phase_block(fc, img_ptr, img_vec, s2p, n_super, kp, k, q0, q1, q2, r2, i2);
  } else {
#pragma unroll
    for (int i = 0; i < 9; ++i) r2[i] = r1[i], i2[i] = i1[i];
  }
  const double w = 0.5 * inv_sqrt_m[k] * inv_sqrt_m[kp];
  const size_t n3 = 3 * (size_t)n_prim;
  double* dq = dyn + (size_t)iq * n3 * n3 * 2;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      // (D + D^H)/2 at (k a, k' b); its conjugate at (k' b, k a).  On the diagonal block the same thread writes
      // both entries of each (a, b) / (b, a) pair, with the same values.
      const double re = w * (r1[a * 3 + b] + r2[b * 3 + a]);
      const double im = w * (i1[a * 3 + b] - i2[b * 3 + a]);
      const size_t u = ((3 * k + a) * n3 + 3 * kp + b) * 2, l = ((3 * kp + b) * n3 + 3 * k + a) * 2;
      dq[u] = re;
      dq[u + 1] = im;
      dq[l] = re;
      dq[l + 1] = -im;
    }
  }
}

}  // namespace
}  // namespace chg

using namespace chg;

extern "C" int chg_dynamical_matrices(const double* fc, const int32_t* img_ptr, const double* img_vec,
                                      const int32_t* s2p, const double* inv_sqrt_m, int32_t n_prim, int32_t n_super,
                                      const double* qpoints, int32_t n_q, double* dyn, void* stream) {
  CHG_CHECK_ARG(n_prim >= 0 && n_super >= 0 && n_q >= 0, "negative size");
  if (n_prim == 0 || n_q == 0) return CHG_OK;
  CHG_CHECK_ARG(fc && img_ptr && img_vec && s2p && inv_sqrt_m && qpoints && dyn, "null pointer");
  CHG_CHECK_ARG((int64_t)n_prim * n_prim < (1ll << 31), "too many primitive atoms");
  const int64_t q_blocks = ((int64_t)n_q + DYN_THREADS - 1) / DYN_THREADS;
  CHG_CHECK_ARG(q_blocks <= 65535, "too many q-points in one call (at most 65535 * 128)");
  const dim3 grid((unsigned)(n_prim * n_prim), (unsigned)q_blocks);
  dynamical_matrices_kernel<<<grid, DYN_THREADS, 0, as_stream(stream)>>>(fc, img_ptr, img_vec, s2p, inv_sqrt_m,
                                                                          n_prim, n_super, qpoints, n_q, dyn);
  CHG_LAUNCH_END();
}
