// chg_linear, warp-specialised wgmma pipeline fed by 2-D TMA tensor maps (k in {64,128},
// no row gather/scatter):   y = x @ wt (+ bias) (+ residual)
//
//   warp 8      producer   one lane issues cp.async.bulk.tensor.2d loads (128B swizzle) of the
//                          next [128 rows x 64 cols] chunk into a 2-stage shared-memory ring
//                          (and of the residual tile into the output stage)
//   warps 0-7   consumers  two warpgroups, rows 0-63 / 64-127 of every tile: each warp reads its
//                          m16 x k8 A fragments from the swizzled stage (conflict-free), splits
//                          them hi/lo (3xTF32) and the warpgroup issues 8 k-steps x 3 split terms
//                          of wgmma.mma_async m64 x NT x k8 per chunk against the weight panel
//                          images (accumulators in registers); then + bias / residual, swizzled
//                          store to the output stage, one lane issues the TMA tensor store
// Every hand-off is an mbarrier (full/empty per ring slot); nothing on the critical path is a
// synchronous global access, so HBM stays busy while the tensor cores work on the current chunk.
#include <cuda.h>

#include "common.cuh"
#include "tc.cuh"

namespace chg {
namespace {

constexpr int NTHR = 288;
constexpr int PRODUCER_WARP = 8;
constexpr int S_IN = 2;                 // input ring depth (chunks of 128 rows x 64 floats)
constexpr int PANEL = 128 * 128;        // bytes of one 128-row x 32-float swizzled panel
constexpr int IN_STAGE = 2 * PANEL;     // 64 columns = 2 panels

struct Bars {
  uint64_t in_full[S_IN], in_empty[S_IN];
  uint64_t res_full, out_empty;
};

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          tc::smem_u32(smem_dst)),
      "l"(map), "r"(tc::smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, int c0, int c1, const void* smem_src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map),
               "r"(tc::smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
// byte offset of 16-byte chunk `c` of row `r` inside a 128B-swizzled panel
__device__ __forceinline__ int swz(int r, int c) { return r * 128 + ((c ^ (r & 7)) << 4); }
// byte offset of element (r, col) of a tile stored as consecutive 32-column swizzled panels
__device__ __forceinline__ int panel_offset(int r, int col) { return (col >> 5) * PANEL + swz(r, (col & 31) >> 2) + (col & 3) * 4; }

template <int NT>
__global__ void __launch_bounds__(NTHR, 1)
linear_ws_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                 const __grid_constant__ CUtensorMap map_r, int m, int k, const float* __restrict__ wt,
                 const float* __restrict__ bias, int has_residual, int n_out) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 128B-swizzled panels must start on 1024-byte boundaries of the shared address space
  uint8_t* s_in = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);  // S_IN x IN_STAGE
  uint8_t* s_out = s_in + S_IN * IN_STAGE;               // NT/32 panels
  uint8_t* s_bhi = s_out + (NT / 32) * PANEL;
  uint8_t* s_blo = s_bhi + (size_t)NT * k * 4;
  __shared__ __align__(8) Bars bars;
  __shared__ __align__(16) float s_bias[NT];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int col_base = blockIdx.y * NT;
  const int n_tiles = (m + 127) / 128;
  const int k_chunks = k / 64;

  // ---- one-time setup: weight images, bias, barriers ------------------------------------------
  {
    const int n4 = NT / 4, total4 = n4 * k;
    for (int i4 = tid; i4 < total4; i4 += NTHR) {
      const int kk = i4 / n4, n0 = (i4 % n4) * 4;
      const float4 v = ldg4(wt + (size_t)kk * n_out + col_base + n0);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        uint32_t hi, lo;
        tc::split_tf32(f4at(v, e), hi, lo);
        const uint32_t off = tc::kmajor_offset(n0 + e, kk, k);
        *reinterpret_cast<uint32_t*>(s_bhi + off) = hi;
        *reinterpret_cast<uint32_t*>(s_blo + off) = lo;
      }
    }
  }
  if (tid < NT) s_bias[tid] = bias != nullptr ? bias[col_base + tid] : 0.f;
  if (tid == 0) {
    for (int i = 0; i < S_IN; ++i) {
      tc::mbar_init(&bars.in_full[i], 1);
      tc::mbar_init(&bars.in_empty[i], 256);
    }
    tc::mbar_init(&bars.res_full, 1);
    tc::mbar_init(&bars.out_empty, 1);
    tc::mbar_fence_init();
  }
  tc::fence_async_smem();
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    // ================= producer =================
    if (lane == 0) {
      int it = 0, tile_it = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tile_it) {
        const int base = tile * 128;
        for (int kc = 0; kc < k_chunks; ++kc, ++it) {
          const int s = it % S_IN;
          tc::mbar_wait(&bars.in_empty[s], ((it / S_IN) & 1) ^ 1);
          tc::mbar_expect_tx(&bars.in_full[s], IN_STAGE);
          tma_load_2d(s_in + s * IN_STAGE, &map_x, kc * 64, base, &bars.in_full[s]);
          tma_load_2d(s_in + s * IN_STAGE + PANEL, &map_x, kc * 64 + 32, base, &bars.in_full[s]);
        }
        if (has_residual) {  // after the inputs, so that waiting for the output stage does not stall them
          tc::mbar_wait(&bars.out_empty, (tile_it & 1) ^ 1);
          tc::mbar_expect_tx(&bars.res_full, (uint32_t)(NT / 32) * PANEL);
#pragma unroll
          for (int p = 0; p < NT / 32; ++p) tma_load_2d(s_out + p * PANEL, &map_r, col_base + p * 32, base, &bars.res_full);
        }
      }
    }
  } else {
    // ================= consumer warpgroups (warps 0..3: rows 0..63, warps 4..7: rows 64..127) =================
    const int t = tid;            // 0..255
    const int row0 = (warp >> 2) * 64;
    const uint32_t bhi_addr = tc::smem_u32(s_bhi), blo_addr = tc::smem_u32(s_blo);
    const uint32_t sbo = (uint32_t)(k / 4) * 128;
    int it = 0, tile_it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tile_it) {
      const int base = tile * 128;
      float acc[NT / 2];
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
      for (int kc = 0; kc < k_chunks; ++kc, ++it) {
        const int s = it % S_IN;
        tc::mbar_wait(&bars.in_full[s], (it / S_IN) & 1);
        const uint8_t* stage = s_in + s * IN_STAGE;
        tc::wg_gemm_k64<NT>(acc, [&](int r, int kk) { return *reinterpret_cast<const float*>(stage + panel_offset(row0 + r, kk)); },
                            bhi_addr + kc * 2048, blo_addr + kc * 2048, sbo);
        tc::mbar_arrive(&bars.in_empty[s]);
      }
      if (has_residual) tc::mbar_wait(&bars.res_full, tile_it & 1);
      tc::wg_barrier(2, 256);  // the previous tile's TMA store has finished reading the output stage
#pragma unroll
      for (int i = 0; i < NT / 2; i += 2) {
        const int r = row0 + tc::frag_row(i), col = tc::frag_col(i);
        float2* dst = reinterpret_cast<float2*>(s_out + panel_offset(r, col));
        float2 o = make_float2(acc[i] + s_bias[col], acc[i + 1] + s_bias[col + 1]);
        if (has_residual) {
          const float2 res = *dst;
          o.x += res.x;
          o.y += res.y;
        }
        *dst = o;
      }
      tc::fence_async_smem();
      tc::wg_barrier(2, 256);
      if (t == 0) {
#pragma unroll
        for (int p = 0; p < NT / 32; ++p) tma_store_2d(&map_y, col_base + p * 32, base, s_out + p * PANEL);
        tc::bulk_commit();
        tc::bulk_wait_read<0>();
        tc::mbar_arrive(&bars.out_empty);
      }
    }
    if (t == 0) tc::bulk_wait_all<0>();
  }
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                             const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                             CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn encode_fn() {
  static EncodeFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(p);
  }
  return fn;
}

// [rows x cols] fp32 row-major matrix, box = 128 rows x 32 floats, 128B swizzle
bool make_map(CUtensorMap* map, const float* ptr, int rows, int cols) {
  EncodeFn fn = encode_fn();
  if (fn == nullptr) return false;
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)cols * 4};
  const cuuint32_t box[2] = {32, 128};
  const cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int NT>
int launch_ws(const CUtensorMap& mx, const CUtensorMap& my, const CUtensorMap& mr, int m, int k, const float* wt,
              const float* bias, int has_residual, int n_out, cudaStream_t stream) {
  const int smem = S_IN * IN_STAGE + (NT / 32) * PANEL + 2 * NT * k * 4 + 1024;
  static int max_smem_set[MAX_DEVICES] = {};  // per device: the attribute belongs to its context
  int& smem_set = max_smem_set[device_ordinal()];
  if (smem > smem_set) {
    CHG_CUDA(cudaFuncSetAttribute(linear_ws_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    smem_set = smem;
  }
  const int n_tiles = (m + 127) / 128;
  const int col_tiles = n_out / NT;
  dim3 grid(min(n_tiles, max(1, sm_count() / col_tiles)), col_tiles);
  linear_ws_kernel<NT><<<grid, NTHR, smem, stream>>>(mx, my, mr, m, k, wt, bias, has_residual, n_out);
  CHG_LAUNCH_END();
}

}  // namespace

// returns 1 if this kernel cannot take the call (caller falls back), else the launch status (<= 0)
int linear_ws(const float* x, int m, int k, const float* wt, const float* bias, const float* residual, int n_out,
              float* y, cudaStream_t stream) {
  if (k != 64 && k != 128) return 1;
  CUtensorMap mx, my, mr;
  if (!make_map(&mx, x, m, k) || !make_map(&my, y, m, n_out)) return 1;
  if (residual != nullptr) {
    if (!make_map(&mr, residual, m, n_out)) return 1;
  } else {
    mr = my;
  }
  if (n_out % 128 == 0 && k == 64) return launch_ws<128>(mx, my, mr, m, k, wt, bias, residual != nullptr, n_out, stream);
  return launch_ws<64>(mx, my, mr, m, k, wt, bias, residual != nullptr, n_out, stream);
}

}  // namespace chg
