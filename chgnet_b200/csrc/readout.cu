// Readout: LayerNorm -> MLP 64->64->..->1 -> per-graph energy sum, fused with its own
// reverse (d sum(E) / d x) and the AtomRef composition sum.
// Reference: chgnet/model/model.py:497-509 (readout_norm, mlp, pooling) and
// composition_model.py:175-205.  One warp per atom; a lane owns features lane, lane+32.
#include "common.cuh"

namespace chg {
namespace {

constexpr int MAX_HIDDEN = 4;

__global__ void __launch_bounds__(256)
readout_kernel(const float* __restrict__ x, const int32_t* __restrict__ z, const int32_t* __restrict__ owner,
               int n_atoms, const float* __restrict__ ln, const float* __restrict__ mlp_wt,
               const float* __restrict__ mlp_w, const float* __restrict__ mlp_b, int n_hidden,
               const float* __restrict__ w_last, float b_last, const float* __restrict__ atom_ref,
               float* __restrict__ site_e, float* __restrict__ h_out, double* __restrict__ e_graph,
               double* __restrict__ e_ref, float* __restrict__ g_x) {
  extern __shared__ __align__(16) float smem[];
  float* s_wt = smem;                          // [L][64][64] k-major
  float* s_w = s_wt + n_hidden * 4096;         // [L][64][64] PyTorch layout (reverse only)
  const bool need_grad = g_x != nullptr;
  for (int i = threadIdx.x; i < n_hidden * 4096; i += blockDim.x) {
    s_wt[i] = mlp_wt[i];
    if (need_grad) s_w[i] = mlp_w[i];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  const float wl0 = w_last[lane], wl1 = w_last[lane + 32];
  for (int atom = warp; atom < n_atoms; atom += n_warps) {
    float h0 = x[(size_t)atom * 64 + lane], h1 = x[(size_t)atom * 64 + lane + 32];
    float xh0 = 0.f, xh1 = 0.f, rstd = 1.f;
    if (ln != nullptr) {
      const float mean = sum32(h0 + h1) * (1.f / 64.f);
      const float d0 = h0 - mean, d1 = h1 - mean;
      const float var = sum32(fmaf(d0, d0, d1 * d1)) * (1.f / 64.f);
      rstd = 1.f / sqrtf(var + 1e-5f);
      xh0 = d0 * rstd;
      xh1 = d1 * rstd;
      h0 = fmaf(xh0, ln[lane], ln[64 + lane]);
      h1 = fmaf(xh1, ln[lane + 32], ln[64 + lane + 32]);
    }
    if (h_out != nullptr) {
      h_out[(size_t)atom * 64 + lane] = h0;
      h_out[(size_t)atom * 64 + lane + 32] = h1;
    }
    float za[MAX_HIDDEN], zb[MAX_HIDDEN];  // pre-activations of each hidden layer
#pragma unroll
    for (int l = 0; l < MAX_HIDDEN; ++l) {
      if (l < n_hidden) {
        const float* wt = s_wt + l * 4096;
        float a = mlp_b[l * 64 + lane], b = mlp_b[l * 64 + lane + 32];
        for (int k = 0; k < 32; ++k) {
          const float v0 = __shfl_sync(0xffffffffu, h0, k), v1 = __shfl_sync(0xffffffffu, h1, k);
          a = fmaf(v0, wt[k * 64 + lane], a);
          b = fmaf(v0, wt[k * 64 + lane + 32], b);
          a = fmaf(v1, wt[(k + 32) * 64 + lane], a);
          b = fmaf(v1, wt[(k + 32) * 64 + lane + 32], b);
        }
        za[l] = a;
        zb[l] = b;
        h0 = silu_f(a);
        h1 = silu_f(b);
      }
    }
    const float se = sum32(fmaf(h0, wl0, h1 * wl1)) + b_last;
    if (lane == 0) {
      site_e[atom] = se;
      const int g = owner[atom];
      atomicAdd(e_graph + g, (double)se);
      {
        const int zi = z[atom] - 1;  // range-checked on the host (IndexError); NaN for raw C-ABI callers
        atomicAdd(e_ref + g, (zi >= 0 && zi < CHG_MAX_Z) ? (double)atom_ref[zi] : (double)__int_as_float(0x7fc00000));
      }
    }
    if (need_grad) {
      // g_h_last = w_last; walk back: g_z = g_h * silu'(z); g_h_prev[k] = sum_n g_z[n] W[n][k]
      float g0 = wl0, g1 = wl1;
#pragma unroll
      for (int l = MAX_HIDDEN - 1; l >= 0; --l) {
        if (l < n_hidden) {
          const float* w = s_w + l * 4096;
          const float gz0 = g0 * dsilu_f(za[l]), gz1 = g1 * dsilu_f(zb[l]);
          float a = 0.f, b = 0.f;
          for (int n = 0; n < 32; ++n) {
            const float v0 = __shfl_sync(0xffffffffu, gz0, n), v1 = __shfl_sync(0xffffffffu, gz1, n);
            a = fmaf(v0, w[n * 64 + lane], a);
            b = fmaf(v0, w[n * 64 + lane + 32], b);
            a = fmaf(v1, w[(n + 32) * 64 + lane], a);
            b = fmaf(v1, w[(n + 32) * 64 + lane + 32], b);
          }
          g0 = a;
          g1 = b;
        }
      }
      if (ln != nullptr) {
        const float gx0 = g0 * ln[lane], gx1 = g1 * ln[lane + 32];
        const float m1 = sum32(gx0 + gx1) * (1.f / 64.f);
        const float m2 = sum32(fmaf(gx0, xh0, gx1 * xh1)) * (1.f / 64.f);
        g0 = rstd * (gx0 - m1 - xh0 * m2);
        g1 = rstd * (gx1 - m1 - xh1 * m2);
      }
      g_x[(size_t)atom * 64 + lane] = g0;
      g_x[(size_t)atom * 64 + lane + 32] = g1;
    }
  }
}

}  // namespace
}  // namespace chg

using namespace chg;

extern "C" int chg_readout(const float* x, const int32_t* z, const int32_t* atom_owner, int32_t n_atoms,
                           const float* ln, const float* mlp_wt, const float* mlp_w, const float* mlp_b,
                           int32_t n_hidden, const float* w_last, float b_last, const float* atom_ref,
                           float* site_e, float* h_out, double* e_graph, double* e_ref, float* g_x, void* stream) {
  CHG_CHECK_ARG(n_atoms >= 0, "negative size");
  CHG_CHECK_ARG(n_hidden >= 1 && n_hidden <= MAX_HIDDEN, "n_hidden must be in [1, 4]");
  if (n_atoms == 0) return CHG_OK;
  CHG_CHECK_ARG(x && z && atom_owner && mlp_wt && mlp_b && w_last && atom_ref && site_e && e_graph && e_ref,
                "null pointer");
  CHG_CHECK_ARG(g_x == nullptr || mlp_w != nullptr, "mlp_w is required when g_x is requested");
  const int smem = 2 * n_hidden * 4096 * 4;
  static int max_smem_set[MAX_DEVICES] = {};  // per device: the attribute belongs to its context
  int& smem_set = max_smem_set[device_ordinal()];
  if (smem > smem_set) {
    CHG_CUDA(cudaFuncSetAttribute(readout_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    smem_set = smem;
  }
  const int blocks = max(1, min((n_atoms + 7) / 8, sm_count() * 2));
  readout_kernel<<<blocks, 256, smem, as_stream(stream)>>>(x, z, atom_owner, n_atoms, ln, mlp_wt, mlp_w, mlp_b,
                                                           n_hidden, w_last, b_last, atom_ref, site_e, h_out,
                                                           e_graph, e_ref, g_x);
  CHG_LAUNCH_END();
}
