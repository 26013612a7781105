// chg_linear on the Hopper tensor cores (wgmma, sm_90a), 3xTF32.
//
//   y[yr] = x[xr] @ wt (+ bias) (+ residual[yr])        x rows of k floats, wt [k][n_out]
//
// One persistent CTA per SM, two warpgroups working on alternating 128-row tiles so that one
// group's loads / epilogue overlap the other group's MMAs.  Per 64-column chunk of k:
//   global rows (64-float chunks, coalesced, with the optional row gather) -> shared staging ->
//   each warp reads its m16 x k8 A fragments from the staging rows, splits them hi / lo ->
//   wgmma.mma_async m64 x NT x k8 (two 64-row blocks, 8 k-steps x 3 split terms; B = the
//   [NT x k] weight panel, resident in shared memory as hi and lo images in the K-major
//   no-swizzle layout), accumulators in registers across the k chunks
// Epilogue: accumulator fragments -> shared staging (32 columns at a time) -> + bias/residual ->
// coalesced global rows (with the optional row scatter).
#include "common.cuh"
#include "tc.cuh"

namespace chg {
namespace {

constexpr int NTHR = 256;

constexpr int IN_LD = 68;   // staging stride (floats) of a 64-float input chunk row: conflict-free fragment reads
constexpr int OUT_LD = 36;  // staging stride of a 32-float output chunk row
constexpr int STAGE_FLOATS = 128 * IN_LD;

template <int NT>
__global__ void __launch_bounds__(NTHR, 1)
linear_tc_kernel(const float* __restrict__ x, const int32_t* __restrict__ x_rows, int m, int k,
                 const float* __restrict__ wt, const float* __restrict__ bias, const float* residual,
                 const int32_t* __restrict__ y_rows, int n_out, float* y) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint8_t* s_bhi = smem_raw;
  uint8_t* s_blo = smem_raw + (size_t)NT * k * 4;
  float* s_stage_all = reinterpret_cast<float*>(smem_raw + (size_t)2 * NT * k * 4);
  __shared__ int s_yrow[2][128];

  const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127;
  const int col_base = blockIdx.y * NT;
  float* stage = s_stage_all + wg * STAGE_FLOATS;

  // weight panel -> hi / lo operand images (element (n, kk) = wt[kk][col_base + n]); float4 loads,
  // all of a thread's loads issued before the first dependent store
  {
    constexpr int PER = 8;  // float4 per thread per round
    const int n4 = NT / 4, total4 = n4 * k;
    for (int base4 = 0; base4 < total4; base4 += NTHR * PER) {
      float4 v[PER];
#pragma unroll
      for (int q = 0; q < PER; ++q) {
        const int i4 = base4 + q * NTHR + tid;
        v[q] = i4 < total4 ? ldg4(wt + (size_t)(i4 / n4) * n_out + col_base + (i4 % n4) * 4)
                           : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int q = 0; q < PER; ++q) {
        const int i4 = base4 + q * NTHR + tid;
        if (i4 < total4) {
          const int kk = i4 / n4, n0 = (i4 % n4) * 4;
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            uint32_t hi, lo;
            tc::split_tf32(f4at(v[q], e), hi, lo);
            const uint32_t off = tc::kmajor_offset(n0 + e, kk, k);
            *reinterpret_cast<uint32_t*>(s_bhi + off) = hi;
            *reinterpret_cast<uint32_t*>(s_blo + off) = lo;
          }
        }
      }
    }
  }
  tc::fence_async_smem();
  __syncthreads();

  const uint32_t bhi_addr = tc::smem_u32(s_bhi), blo_addr = tc::smem_u32(s_blo);
  const uint32_t sbo = (uint32_t)(k / 4) * 128;
  const int bar_id = 1 + wg;

  const int n_tiles = (m + 127) / 128;
  const int c4_in = t & 15, row0_in = t >> 4;
  for (int tile = blockIdx.x * 2 + wg; tile < n_tiles; tile += gridDim.x * 2) {
    const int base = tile * 128;
    {
      const int r = min(base + t, m - 1);
      s_yrow[wg][t] = (base + t < m) ? (y_rows != nullptr ? __ldg(y_rows + r) : r) : -1;
    }
    float acc[2][NT / 2];
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) acc[mb][i] = 0.f;

    for (int kc = 0; kc < k; kc += 64) {
      float4 v[16];
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        const int r = min(base + row0_in + q * 8, m - 1);
        const int xr = x_rows != nullptr ? __ldg(x_rows + r) : r;
        v[q] = ldg4(x + (size_t)xr * k + kc + c4_in * 4);
      }
#pragma unroll
      for (int q = 0; q < 16; ++q) sts4(stage + (row0_in + q * 8) * IN_LD + c4_in * 4, v[q]);
      tc::wg_barrier(bar_id, 128);
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
        const float* a_rows = stage + mb * 64 * IN_LD;
        tc::wg_gemm_k64<NT>(acc[mb], [&](int r, int kk) { return a_rows[r * IN_LD + kk]; }, bhi_addr + kc * 32,
                            blo_addr + kc * 32, sbo);
      }
      tc::wg_barrier(bar_id, 128);  // the staging rows may be overwritten
    }

    // accumulator fragments -> staging (32 columns at a time) -> coalesced global rows
#pragma unroll
    for (int c = 0; c < NT; c += 32) {
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int i = c / 2; i < c / 2 + 16; i += 2)
          *reinterpret_cast<float2*>(stage + (mb * 64 + tc::frag_row(i)) * OUT_LD + tc::frag_col(i) - c) =
              make_float2(acc[mb][i], acc[mb][i + 1]);
      tc::wg_barrier(bar_id, 128);
      {
        const int c4 = t & 7, row0 = t >> 3;
        const int col = col_base + c + c4 * 4;
        int orow[8];
        float4 o[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) orow[q] = s_yrow[wg][row0 + q * 16];
        float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (bias != nullptr) b4 = ldg4(bias + col);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          o[q] = b4;
          if (residual != nullptr && orow[q] >= 0)
            o[q] = o[q] + *reinterpret_cast<const float4*>(residual + (size_t)orow[q] * n_out + col);
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) o[q] = o[q] + lds4(stage + (row0 + q * 16) * OUT_LD + c4 * 4);
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (orow[q] >= 0) stg4(y + (size_t)orow[q] * n_out + col, o[q]);
      }
      tc::wg_barrier(bar_id, 128);
    }
  }
}

template <int NT>
int launch_linear_tc(const float* x, const int32_t* x_rows, int m, int k, const float* wt, const float* bias,
                     const float* residual, const int32_t* y_rows, int n_out, float* y, cudaStream_t stream) {
  const int smem = 2 * NT * k * 4 + 2 * STAGE_FLOATS * 4;
  static int max_smem_set[MAX_DEVICES] = {};  // per device: the attribute belongs to its context
  int& smem_set = max_smem_set[device_ordinal()];
  if (smem > smem_set) {
    CHG_CUDA(cudaFuncSetAttribute(linear_tc_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    smem_set = smem;
  }
  const int n_tiles = (m + 127) / 128;
  const int col_tiles = n_out / NT;
  const int per_col = max(1, sm_count() / col_tiles);
  dim3 grid(min((n_tiles + 1) / 2, per_col), col_tiles);
  linear_tc_kernel<NT><<<grid, NTHR, smem, stream>>>(x, x_rows, m, k, wt, bias, residual, y_rows, n_out, y);
  CHG_LAUNCH_END();
}

}  // namespace

int linear_tc(const float* x, const int32_t* x_rows, int m, int k, const float* wt, const float* bias,
              const float* residual, const int32_t* y_rows, int n_out, float* y, cudaStream_t stream) {
  if (n_out % 128 == 0 && k <= 128)
    return launch_linear_tc<128>(x, x_rows, m, k, wt, bias, residual, y_rows, n_out, y, stream);
  return launch_linear_tc<64>(x, x_rows, m, k, wt, bias, residual, y_rows, n_out, y, stream);
}

}  // namespace chg
