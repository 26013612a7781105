// AtomConv / BondConv message kernels on the Hopper tensor cores (wgmma, sm_90a): forward and reverse.
//
// Same entry points, arguments and arithmetic as the FFMA kernels in gated.cu; the two
// 64x64 second-layer products of the GatedMLP (and their transposes in the reverse) run on
// the tensor cores as 3xTF32 (tc.cuh) with accumulators in registers:
//
//   (a) cooperative phase, 16 lanes x float4 per 64-wide half-row (coalesced): gather + add
//       the pre-activation rows, SiLU, write the 128-row tile to shared memory
//   (b) each warp reads the A fragments of its rows from the tile, splits hi/lo, and the
//       warpgroup issues 8 x 3 wgmma.mma_async m64n64k8 per (64-row block, half) against the
//       weight images resident in shared memory (core half, then gate half)
//   (c) the accumulator fragments overwrite the rows they were computed from
//   (d) cooperative epilogue in the same 16-lane layout as the FFMA kernel: bias, LayerNorm
//       (shfl reductions), SiLU x sigmoid, bond-weight smoothing, coalesced stores
//
// One persistent CTA per SM = two warpgroups on alternating 128-row tiles (one group's
// gathers / epilogue overlap the other's MMAs).
// Shared memory: 4 weight images (64 KB) + 2 x [128][132] fp32 tiles (132 KB).
#include "gated_common.cuh"
#include "tc.cuh"

namespace chg {
namespace gated {
namespace {

constexpr int NTHR = 256;
constexpr int TMT = 128;             // rows per warpgroup tile
constexpr int IMG = 64 * 64 * 4;     // bytes of one 64x64 operand image
constexpr int STAGE_FLOATS = TMT * HS;

struct SmemLayout {
  static constexpr int IMG_OFF = 0;                                // Bc_hi, Bc_lo, Bg_hi, Bg_lo
  static constexpr int STAGE_OFF = 4 * IMG;                        // 2 x [128][HS] floats
  static constexpr int B2_OFF = STAGE_OFF + 2 * STAGE_FLOATS * 4;  // 128 floats
  static constexpr int LN_OFF = B2_OFF + 128 * 4;                  // 256 floats
  static constexpr int IDX_OFF = LN_OFF + 256 * 4;                 // 2 x 3 x 128 ints
  static constexpr int TOTAL = IDX_OFF + 2 * 3 * TMT * 4;
};

// image element (n, kk) = src[kk * ld + col0 + n]   (64 x 64, K-major, no swizzle)
__device__ __forceinline__ void build_image(uint8_t* hi, uint8_t* lo, const float* __restrict__ src, int ld,
                                            int col0, int tid) {
  for (int i = tid; i < 4096; i += NTHR) {
    const int kk = i >> 6, n = i & 63;
    uint32_t h, l;
    tc::split_tf32(__ldg(src + (size_t)kk * ld + col0 + n), h, l);
    const uint32_t off = tc::kmajor_offset(n, kk, 64);
    *reinterpret_cast<uint32_t*>(hi + off) = h;
    *reinterpret_cast<uint32_t*>(lo + off) = l;
  }
}

// stage row r [0:64 | 64:128] x (Bc | Bg) -> the same row of the stage [0:64 | 64:128], all 128 threads of the
// warpgroup; each warp only reads and rewrites its own 16-row slices, so no barrier is needed in between
__device__ __forceinline__ void tile_blockdiag_mma(float* stage, uint32_t img_addr) {
#pragma unroll 1
  for (int half = 0; half < 2; ++half) {
    const uint32_t bhi = img_addr + half * 2 * IMG, blo = bhi + IMG;
#pragma unroll 1
    for (int mb = 0; mb < 2; ++mb) {
      float* rows = stage + mb * 64 * HS + half * 64;
      float d[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) d[i] = 0.f;
      tc::wg_gemm_k64<64>(d, [&](int r, int k) { return rows[r * HS + k]; }, bhi, blo, 2048);
#pragma unroll
      for (int i = 0; i < 32; i += 2)
        *reinterpret_cast<float2*>(rows + tc::frag_row(i) * HS + tc::frag_col(i)) = make_float2(d[i], d[i + 1]);
    }
  }
}

// ------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(NTHR, 1) gated_fwd_tc_kernel(const FwdArgs a) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint8_t* s_img = smem_raw + SmemLayout::IMG_OFF;
  float* s_b2 = reinterpret_cast<float*>(smem_raw + SmemLayout::B2_OFF);
  float* s_ln = reinterpret_cast<float*>(smem_raw + SmemLayout::LN_OFF);

  const int tid = threadIdx.x;
  const bool use_ln = a.ln != nullptr;
  build_image(s_img, s_img + IMG, a.w2t, 128, 0, tid);             // core: (n=c, kk=k) = w2t[k][c]
  build_image(s_img + 2 * IMG, s_img + 3 * IMG, a.w2t, 128, 64, tid);  // gate
  if (tid < 128) s_b2[tid] = a.b2[tid];
  if (use_ln) s_ln[tid] = a.ln[tid];
  tc::fence_async_smem();
  __syncthreads();

  const int wg = tid >> 7, t = tid & 127, bar_id = 1 + wg;
  const uint32_t img_addr = tc::smem_u32(s_img);
  float* stage = reinterpret_cast<float*>(smem_raw + SmemLayout::STAGE_OFF) + wg * STAGE_FLOATS;
  int* s_idx = reinterpret_cast<int*>(smem_raw + SmemLayout::IDX_OFF) + wg * 3 * TMT;
  const int tx = t & 15, ty = t >> 4;  // 16 lanes per row, 8 row groups
  const int c0 = tx * 4;

  const int n_tiles = (a.n_rows + TMT - 1) / TMT;
  for (int tile = blockIdx.x * 2 + wg; tile < n_tiles; tile += gridDim.x * 2) {
    const int base = tile * TMT;
    {
      const int r = min(base + t, a.n_rows - 1);
      s_idx[t] = a.idx0[r];
      s_idx[TMT + t] = a.idx1[r];
      s_idx[2 * TMT + t] = a.idx2[r];
    }
    tc::wg_barrier(bar_id, 128);

    // (a) gather + add the pre-activation rows, SiLU -> stage
#pragma unroll 1
    for (int it = 0; it < 4; ++it) {
      const int r0 = it * 32 + ty * 4;
      float acc[4][8];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
      gather_pre<TMT>(acc, a.p_a, a.p_b, a.p_c, s_idx, base, a.n_rows, r0, c0);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int g = base + r0 + i;
        if (a.save_pre != nullptr && g < a.n_rows) {
          stg4(a.save_pre + (size_t)g * 128 + c0, make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]));
          stg4(a.save_pre + (size_t)g * 128 + 64 + c0, make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]));
        }
        sts4(stage + (r0 + i) * HS + c0,
             make_float4(silu_f(acc[i][0]), silu_f(acc[i][1]), silu_f(acc[i][2]), silu_f(acc[i][3])));
        sts4(stage + (r0 + i) * HS + 64 + c0,
             make_float4(silu_f(acc[i][4]), silu_f(acc[i][5]), silu_f(acc[i][6]), silu_f(acc[i][7])));
      }
    }
    tc::wg_barrier(bar_id, 128);

    // (b) second layer on the tensor cores, (c) accumulators back to shared memory
    tile_blockdiag_mma(stage, img_addr);
    tc::wg_barrier(bar_id, 128);

    // (d) epilogue: + b2 -> LayerNorm -> silu * sigmoid -> smoothing -> store
    float4 g1, b1, g2, b2v;
    if (use_ln) {
      g1 = lds4(s_ln + c0);
      b1 = lds4(s_ln + 64 + c0);
      g2 = lds4(s_ln + 128 + c0);
      b2v = lds4(s_ln + 192 + c0);
    }
    const float4 bc = lds4(s_b2 + c0), bg = lds4(s_b2 + 64 + c0);
#pragma unroll 1
    for (int it = 0; it < 4; ++it) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = it * 32 + ty * 4 + i;
        const int g = base + row;
        const bool valid = g < a.n_rows;
        const float4 pc = lds4(stage + row * HS + c0) + bc;
        const float4 pg = lds4(stage + row * HS + 64 + c0) + bg;
        if (a.save_p != nullptr && valid) {
          stg4(a.save_p + (size_t)g * 128 + c0, pc);
          stg4(a.save_p + (size_t)g * 128 + 64 + c0, pg);
        }
        float y1[4] = {pc.x, pc.y, pc.z, pc.w};
        float y2[4] = {pg.x, pg.y, pg.z, pg.w};
        if (use_ln) {
          float xh[4], rstd;
          ln_stats(y1, xh, rstd);
#pragma unroll
          for (int j = 0; j < 4; ++j) y1[j] = fmaf(xh[j], f4at(g1, j), f4at(b1, j));
          ln_stats(y2, xh, rstd);
#pragma unroll
          for (int j = 0; j < 4; ++j) y2[j] = fmaf(xh[j], f4at(g2, j), f4at(b2v, j));
        }
        float4 o;
#pragma unroll
        for (int j = 0; j < 4; ++j) f4at(o, j) = silu_f(y1[j]) * sigmoid_f(y2[j]);
        if (MODE == ATOM) {
          o = o * ldg4(a.wgt + (size_t)s_idx[2 * TMT + row] * 64 + c0);
        } else {
          o = o * ldg4(a.wgt + (size_t)s_idx[row] * 64 + c0) * ldg4(a.wgt + (size_t)s_idx[TMT + row] * 64 + c0);
        }
        if (valid) stg4(a.out + (size_t)g * 64 + c0, o);
      }
    }
    tc::wg_barrier(bar_id, 128);  // stage / s_idx are free for the next tile
  }
}

// ------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(NTHR, 1) gated_bwd_tc_kernel(const BwdArgs a) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint8_t* s_img = smem_raw + SmemLayout::IMG_OFF;
  float* s_ln = reinterpret_cast<float*>(smem_raw + SmemLayout::LN_OFF);

  const int tid = threadIdx.x;
  const bool use_ln = a.ln != nullptr;
  // g_h[k] = sum_c g_p[c] W2[c][k]: image element (n=k, kk=c) = w2[c][k]
  build_image(s_img, s_img + IMG, a.w2, 64, 0, tid);
  build_image(s_img + 2 * IMG, s_img + 3 * IMG, a.w2 + 64 * 64, 64, 0, tid);
  if (use_ln) s_ln[tid] = a.ln[tid];
  tc::fence_async_smem();
  __syncthreads();

  const int wg = tid >> 7, t = tid & 127, bar_id = 1 + wg;
  const uint32_t img_addr = tc::smem_u32(s_img);
  float* stage = reinterpret_cast<float*>(smem_raw + SmemLayout::STAGE_OFF) + wg * STAGE_FLOATS;
  int* s_idx = reinterpret_cast<int*>(smem_raw + SmemLayout::IDX_OFF) + wg * 3 * TMT;
  const int tx = t & 15, ty = t >> 4;
  const int c0 = tx * 4;

  const int n_tiles = (a.n_rows + TMT - 1) / TMT;
  for (int tile = blockIdx.x * 2 + wg; tile < n_tiles; tile += gridDim.x * 2) {
    const int base = tile * TMT;
    {
      const int r = min(base + t, a.n_rows - 1);
      s_idx[t] = a.idx0[r];
      s_idx[TMT + t] = a.idx1[r];
      if (MODE == ATOM) s_idx[2 * TMT + t] = a.idx2[r];
    }
    tc::wg_barrier(bar_id, 128);

    // (a) recompute the gate from saved p, bond-weight gradients, LayerNorm reverse -> g_p -> stage
    float4 g1, g2, b1, b2v;
    if (use_ln) {
      g1 = lds4(s_ln + c0);
      b1 = lds4(s_ln + 64 + c0);
      g2 = lds4(s_ln + 128 + c0);
      b2v = lds4(s_ln + 192 + c0);
    }
#pragma unroll 1
    for (int it = 0; it < 4; ++it) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = it * 32 + ty * 4 + i;
        const int g = base + row;
        const bool valid = g < a.n_rows;
        const int r = min(g, a.n_rows - 1);
        const float4 pc4 = ldg4(a.save_p + (size_t)r * 128 + c0);
        const float4 pg4 = ldg4(a.save_p + (size_t)r * 128 + 64 + c0);
        float y1[4] = {pc4.x, pc4.y, pc4.z, pc4.w};
        float y2[4] = {pg4.x, pg4.y, pg4.z, pg4.w};
        float xh1[4], xh2[4], rstd1 = 1.f, rstd2 = 1.f;
        if (use_ln) {
          ln_stats(y1, xh1, rstd1);
          ln_stats(y2, xh2, rstd2);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            y1[j] = fmaf(xh1[j], f4at(g1, j), f4at(b1, j));
            y2[j] = fmaf(xh2[j], f4at(g2, j), f4at(b2v, j));
          }
        }
        float s1[4], core[4], gate[4];
        float4 o;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          s1[j] = sigmoid_f(y1[j]);
          core[j] = y1[j] * s1[j];
          gate[j] = sigmoid_f(y2[j]);
          f4at(o, j) = core[j] * gate[j];
        }
        float4 go;
        if (MODE == ATOM) {
          const float4 gm = ldg4(a.g_in + (size_t)s_idx[row] * 64 + c0);
          const float4 w = ldg4(a.wgt + (size_t)s_idx[2 * TMT + row] * 64 + c0);
          if (valid) stg4(a.g_w0 + (size_t)g * 64 + c0, gm * o);
          go = gm * w;
        } else {
          const float4 gm = ldg4(a.g_in + (size_t)s_idx[row] * 64 + c0);
          const float4 wi = ldg4(a.wgt + (size_t)s_idx[row] * 64 + c0);
          const float4 wj = ldg4(a.wgt + (size_t)s_idx[TMT + row] * 64 + c0);
          const float4 gmo = gm * o;
          if (valid) {
            stg4(a.g_w0 + (size_t)g * 64 + c0, gmo * wj);
            stg4(a.g_w1 + (size_t)g * 64 + c0, gmo * wi);
          }
          go = gm * wi * wj;
        }
        float gy1[4], gy2[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float gj = f4at(go, j);
          gy1[j] = gj * gate[j] * (s1[j] * fmaf(y1[j], 1.f - s1[j], 1.f));
          gy2[j] = gj * core[j] * gate[j] * (1.f - gate[j]);
        }
        if (use_ln) {
          float gx[4], sa = 0.f, sb = 0.f;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            gx[j] = gy1[j] * f4at(g1, j);
            sa += gx[j];
            sb = fmaf(gx[j], xh1[j], sb);
          }
          sa = sum16(sa) * (1.f / 64.f);
          sb = sum16(sb) * (1.f / 64.f);
#pragma unroll
          for (int j = 0; j < 4; ++j) gy1[j] = rstd1 * (gx[j] - sa - xh1[j] * sb);
          sa = 0.f, sb = 0.f;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            gx[j] = gy2[j] * f4at(g2, j);
            sa += gx[j];
            sb = fmaf(gx[j], xh2[j], sb);
          }
          sa = sum16(sa) * (1.f / 64.f);
          sb = sum16(sb) * (1.f / 64.f);
#pragma unroll
          for (int j = 0; j < 4; ++j) gy2[j] = rstd2 * (gx[j] - sa - xh2[j] * sb);
        }
        sts4(stage + row * HS + c0, make_float4(gy1[0], gy1[1], gy1[2], gy1[3]));
        sts4(stage + row * HS + 64 + c0, make_float4(gy2[0], gy2[1], gy2[2], gy2[3]));
      }
    }
    tc::wg_barrier(bar_id, 128);

    // (b) g_h = g_p . W2 on the tensor cores, (c) back to shared memory
    tile_blockdiag_mma(stage, img_addr);
    tc::wg_barrier(bar_id, 128);

    // (d) g_pre = g_h * silu'(pre)
#pragma unroll 1
    for (int it = 0; it < 4; ++it) {
      const int r0 = it * 32 + ty * 4;
      float pre[4][8];
      if (MODE == ATOM) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) pre[i][j] = 0.f;
        gather_pre<TMT>(pre, a.p_a, a.p_b, nullptr, s_idx, base, a.n_rows, r0, c0);
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = min(base + r0 + i, a.n_rows - 1);
          const float4 vc = ldg4(a.save_pre + (size_t)r * 128 + c0);
          const float4 vg = ldg4(a.save_pre + (size_t)r * 128 + 64 + c0);
          pre[i][0] = vc.x; pre[i][1] = vc.y; pre[i][2] = vc.z; pre[i][3] = vc.w;
          pre[i][4] = vg.x; pre[i][5] = vg.y; pre[i][6] = vg.z; pre[i][7] = vg.w;
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int g = base + r0 + i;
        const float4 hc = lds4(stage + (r0 + i) * HS + c0);
        const float4 hg = lds4(stage + (r0 + i) * HS + 64 + c0);
        if (g < a.n_rows) {
          stg4(a.g_pre + (size_t)g * 128 + c0,
               make_float4(hc.x * dsilu_f(pre[i][0]), hc.y * dsilu_f(pre[i][1]), hc.z * dsilu_f(pre[i][2]),
                           hc.w * dsilu_f(pre[i][3])));
          stg4(a.g_pre + (size_t)g * 128 + 64 + c0,
               make_float4(hg.x * dsilu_f(pre[i][4]), hg.y * dsilu_f(pre[i][5]), hg.z * dsilu_f(pre[i][6]),
                           hg.w * dsilu_f(pre[i][7])));
        }
      }
    }
    tc::wg_barrier(bar_id, 128);
  }
}

template <typename KernelT, typename ArgsT>
int launch_tc(KernelT kernel, const ArgsT& a, cudaStream_t stream) {
  if (a.n_rows == 0) return CHG_OK;
  CHG_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemLayout::TOTAL));
  const int n_tiles = (a.n_rows + TMT - 1) / TMT;
  kernel<<<max(1, min((n_tiles + 1) / 2, sm_count())), NTHR, SmemLayout::TOTAL, stream>>>(a);
  CHG_LAUNCH_END();
}

}  // namespace

int atom_conv_fwd_tc(const FwdArgs& a, cudaStream_t stream) { return launch_tc(gated_fwd_tc_kernel<ATOM>, a, stream); }
int bond_conv_fwd_tc(const FwdArgs& a, cudaStream_t stream) { return launch_tc(gated_fwd_tc_kernel<BOND>, a, stream); }
int atom_conv_bwd_tc(const BwdArgs& a, cudaStream_t stream) { return launch_tc(gated_bwd_tc_kernel<ATOM>, a, stream); }
int bond_conv_bwd_tc(const BwdArgs& a, cudaStream_t stream) { return launch_tc(gated_bwd_tc_kernel<BOND>, a, stream); }

}  // namespace gated
}  // namespace chg
