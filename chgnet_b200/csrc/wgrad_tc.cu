// chg_wgrad on the Hopper tensor cores (wgmma, sm_90a):  out[64][n] = act(X[xr])^T . G[gr]   (reduction over the m rows)
//
// The weight gradients of the training step (reference trainer.py:409 loss.backward(): dL/dW of every dense layer) are
// true GEMMs with the ROWS as the contraction dimension: [64 x m] . [m x n], m up to the number of angles (4e5 per GPU in
// the fine-tuning config).  Round 1 ran them on the FFMA pipe (31 TFLOP/s, 25 % of the step).  Here:
//
//   D[j][i] (+)= sum_k G[k][c0 + j] * act(X)[k][i]          A = G^T block (M = 128 columns of G, zero rows when the
//                                                            block is 64 wide), B = act(X)^T (N = 64), K = rows
//
// as 3xTF32 wgmma.mma_async m64n64k8 with BOTH operands in shared memory (warpgroup w takes the 64 columns 64w.. of
// the G block): every 32-row stage is transposed into the no-swizzle K-major operand images (hi and lo parts) by the
// 8 warps - lane <-> column, four rows per 16-byte store, conflict-free - while the MMAs of the previous stage run
// (two stages; wgmma.wait_group 1 before a stage is rewritten).  Accumulator: 32 registers per thread.  Each CTA owns a contiguous range of rows and one 128-column block and writes a
// partial [64][n] tile; the fp64 second pass of train.cu (wgrad_reduce_kernel) sums the partials in fixed order.
#include "common.cuh"
#include "tc.cuh"

namespace chg {

// train.cu
void wgrad_reduce_launch(const float* partial, const float* cs_partial, int n_chunks, int n, float* out, int ldo, float* colsum,
                         cudaStream_t stream);

namespace {

constexpr int WT_THREADS = 256;
constexpr int WT_K = 32;                       // rows per stage
constexpr int A_IMG = 128 * WT_K * 4;          // 16 KB: G^T block, hi or lo
constexpr int B_IMG = 64 * WT_K * 4;           // 8 KB: act(X)^T, hi or lo
constexpr int STAGE = 2 * A_IMG + 2 * B_IMG;   // 48 KB: two stages per CTA, two CTAs per SM
constexpr int WT_PER = WT_K / 32;              // row-quads per warp and column group (8 warps x 4 rows = 32 rows)
constexpr int WT_SMEM = 2 * STAGE + 2 * WT_K * 4 * 2 + 1024;

// ACT: 0 x, 1 silu(x), 2 silu'(x) * x2;  GG = 32-column groups of the G block (2: 64 columns, 4: 128 columns)
template <int ACT, int GG>
__global__ void __launch_bounds__(WT_THREADS, 2)
wgrad_tc_kernel(const float* __restrict__ x, const float* __restrict__ x2, int ldx, const int32_t* __restrict__ x_rows,
                const float* __restrict__ g, int ldg, const int32_t* __restrict__ g_rows, int m, int n, int n_block,
                float* __restrict__ partial, float* __restrict__ cs_partial) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* s_stage = smem_raw;
  int* s_xi = reinterpret_cast<int*>(smem_raw + 2 * STAGE);  // [2][WT_K] row of X
  int* s_gi = s_xi + 2 * WT_K;                               // [2][WT_K] row of G
  __shared__ float s_cs[8][128];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int col_base = blockIdx.y * 128;
  const int n_chunks = gridDim.x;
  const int steps_total = (m + WT_K - 1) / WT_K;
  const int s_beg = (int)((long long)steps_total * blockIdx.x / n_chunks);
  const int s_end = (int)((long long)steps_total * (blockIdx.x + 1) / n_chunks);

  // zero the A images once when the column block is narrower than 128: rows n_block..127 stay zero
  if (n_block < 128) {
    for (int i = tid * 4; i < 2 * STAGE / 4; i += WT_THREADS * 4) sts4(reinterpret_cast<float*>(s_stage) + i, make_float4(0.f, 0.f, 0.f, 0.f));
  }
  __syncthreads();
  const int wg = warp >> 2;
  const bool wg_live = wg == 0 || n_block > 64;  // a 64-wide block leaves the second warpgroup's rows of A zero
  float d[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) d[i] = 0.f;

  float cs[4] = {0.f, 0.f, 0.f, 0.f};  // column sums of G for this lane's columns lane + 32 c
  int it = 0;
  for (int step = s_beg; step < s_end; ++step, ++it) {
    const int st = it & 1;
    uint8_t* a_hi = s_stage + st * STAGE;
    uint8_t* a_lo = a_hi + A_IMG;
    uint8_t* b_hi = a_lo + A_IMG;
    uint8_t* b_lo = b_hi + B_IMG;
    // the MMAs that read this stage two iterations ago have completed (both warpgroups: the barrier below)
    tc::wgmma_wait<1>();
    const int base = step * WT_K;
    if (tid < WT_K) {
      const int row = min(base + tid, m - 1);
      s_xi[st * WT_K + tid] = x_rows != nullptr ? x_rows[row] : row;
      s_gi[st * WT_K + tid] = g_rows != nullptr ? g_rows[row] : row;
    }
    __syncthreads();
    // ---- transpose this stage into the operand images: a work item = (4 consecutive rows, 32 consecutive columns); a warp
    // owns row-quad warp (+ 8 for the second quad of a 64-row stage) of every column group (G block first, then the two
    // feature groups of X).  ALL loads of the stage are issued before the first use (WT_PER (GG + 2) x 4 independent 4-byte
    // loads per thread in flight; two CTAs per SM alternate between loading and transposing).
    constexpr int ITEMS = WT_PER * (GG + 2);
    float v[ITEMS][4], w2[ACT == 2 ? 2 * WT_PER : 1][4];
#pragma unroll
    for (int t = 0; t < ITEMS; ++t) {
      const int quad = warp + 8 * (t % WT_PER), grp = t / WT_PER;
      const bool is_g = grp < GG;
      const int col = (is_g ? grp : grp - GG) * 32 + lane;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int k = quad * 4 + q;
        const bool live = base + k < m;
        if (is_g) {
          v[t][q] = live ? __ldg(g + (size_t)s_gi[st * WT_K + k] * ldg + col_base + col) : 0.f;
        } else {
          v[t][q] = live ? __ldg(x + (size_t)s_xi[st * WT_K + k] * ldx + col) : 0.f;
          if (ACT == 2) w2[t - WT_PER * GG][q] = live ? __ldg(x2 + (size_t)s_xi[st * WT_K + k] * ldx + col) : 0.f;
        }
      }
    }
#pragma unroll
    for (int t = 0; t < ITEMS; ++t) {
      const int quad = warp + 8 * (t % WT_PER), grp = t / WT_PER;
      const bool is_g = grp < GG;
      const int col = (is_g ? grp : grp - GG) * 32 + lane;
      if (is_g) {
        cs[grp < 4 ? grp : 0] += (v[t][0] + v[t][1]) + (v[t][2] + v[t][3]);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (ACT == 1) v[t][q] = silu_f(v[t][q]);
          if (ACT == 2) v[t][q] = dsilu_f(v[t][q]) * w2[t - WT_PER * GG][q];
        }
      }
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) tc::split_tf32(v[t][q], hi[q], lo[q]);
      const uint32_t off = tc::kmajor_offset(col, quad * 4, WT_K);  // 16 bytes: k = 4 quad .. 4 quad + 3 of row `col`
      *reinterpret_cast<uint4*>((is_g ? a_hi : b_hi) + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
      *reinterpret_cast<uint4*>((is_g ? a_lo : b_lo) + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
    tc::fence_async_smem();  // generic-proxy writes -> visible to the tensor core's operand reads
    __syncthreads();
    if (wg_live) {
      // this warpgroup's 64 rows of the G^T image (8192 bytes per 64 rows of a 32-wide K-major image)
      const uint32_t ah = tc::smem_u32(a_hi) + wg * 8192, al = tc::smem_u32(a_lo) + wg * 8192;
      const uint32_t bh = tc::smem_u32(b_hi), bl = tc::smem_u32(b_lo);
      const uint32_t sbo = (WT_K / 4) * 128;
      tc::wgmma_fence();
#pragma unroll
      for (int j = 0; j < WT_K / 8; ++j) {
        const uint64_t dah = tc::smem_desc_kmajor(ah + j * 256, 128, sbo), dal = tc::smem_desc_kmajor(al + j * 256, 128, sbo);
        const uint64_t dbh = tc::smem_desc_kmajor(bh + j * 256, 128, sbo), dbl = tc::smem_desc_kmajor(bl + j * 256, 128, sbo);
        tc::wgmma_tf32_ss_m64n64(d, dah, dbh);
        tc::wgmma_tf32_ss_m64n64(d, dal, dbh);
        tc::wgmma_tf32_ss_m64n64(d, dah, dbl);
      }
      tc::wgmma_commit();
    }
  }
  // ---- wait for the last MMAs, then accumulator fragments -> partial tile: out[i][j], i = feature of X, j = column of G
  tc::wgmma_wait<0>();
  float* dst = partial + (size_t)blockIdx.x * 64 * n;
#pragma unroll
  for (int q = 0; q < 32; ++q) {
    const int j = wg * 64 + tc::frag_row(q);
    if (j < n_block) dst[(size_t)tc::frag_col(q) * n + col_base + j] = d[q];
  }
  if (cs_partial != nullptr) {
#pragma unroll
    for (int c = 0; c < 4; ++c) s_cs[warp][c * 32 + lane] = cs[c];
    __syncthreads();
    if (tid < n_block) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += s_cs[w][tid];
      cs_partial[(size_t)blockIdx.x * n + col_base + tid] = t;
    }
  }
}

}  // namespace

// returns 1 when this kernel does not take the call (caller uses the FFMA kernel)
int wgrad_tc(const float* x, const float* x2, int ldx, const int32_t* x_rows, int x_silu, const float* g, int ldg,
             const int32_t* g_rows, int m, int n_out, float* out, int ldo, float* colsum, float* workspace, int max_chunks,
             cudaStream_t stream) {
  if (m < 4096) return 1;  // small reductions: launch + transposition overhead dominates
  const int n_block = n_out >= 128 ? 128 : 64;
  if (n_out % n_block != 0) return 1;
  const int col_blocks = n_out / n_block;
  const int steps = (m + WT_K - 1) / WT_K;
  int n_chunks = 2 * sm_count() / col_blocks;  // two CTAs per SM
  n_chunks = max(1, min(min(n_chunks, steps), max_chunks));
  float* partial = workspace;
  float* cs_partial = colsum != nullptr ? workspace + (size_t)n_chunks * 64 * n_out : nullptr;
  dim3 grid(n_chunks, col_blocks);
#define CHG_WT(ACT_, GG_)                                                                                                   \
  do {                                                                                                                      \
    static bool attr[MAX_DEVICES] = {}; /* per device: the attribute belongs to its context */                            \
    bool& set = attr[device_ordinal()];                                                                                     \
    if (!set) {                                                                                                             \
      CHG_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<ACT_, GG_>, cudaFuncAttributeMaxDynamicSharedMemorySize, WT_SMEM));      \
      set = true;                                                                                                           \
    }                                                                                                                       \
    wgrad_tc_kernel<ACT_, GG_><<<grid, WT_THREADS, WT_SMEM, stream>>>(x, x2, ldx, x_rows, g, ldg, g_rows, m, n_out, n_block, \
                                                                      partial, cs_partial);                                 \
  } while (0)
  if (n_block == 128) {
    if (x2 != nullptr) CHG_WT(2, 4);
    else if (x_silu) CHG_WT(1, 4);
    else CHG_WT(0, 4);
  } else {
    if (x2 != nullptr) CHG_WT(2, 2);
    else if (x_silu) CHG_WT(1, 2);
    else CHG_WT(0, 2);
  }
#undef CHG_WT
  {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      set_error("chg_wgrad (wgmma): launch failed: %s", cudaGetErrorString(e));
      return CHG_ERR_CUDA;
    }
    count_launch();
  }
  wgrad_reduce_launch(partial, cs_partial, n_chunks, n_out, out, ldo, colsum, stream);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("chg_wgrad (wgmma): reduce launch failed: %s", cudaGetErrorString(e));
    return CHG_ERR_CUDA;
  }
  count_launch();
  return CHG_OK;
}

}  // namespace chg
