// AtomConv / BondConv message + aggregation as ONE warp-specialised wgmma kernel (sm_90a).
//
//   agg[s] = sum_{rows r of segment s} GatedMLP(pre_r) * w_r          (reference layers.py:113-126, 238-254)
//
// with pre_r = the gather-add of 3 (AtomConv) / 4 (BondConv) first-layer rows (DESIGN.md §3.1), the two
// 64x64 second-layer products on the tensor cores (3xTF32, accumulators in registers), LayerNorm +
// SiLU x sigmoid in the epilogue, and the segmented reduction over the centre-sorted (bond-i-sorted) rows done
// inside the CTA: the [rows, 64] message never goes to HBM.
//
// One persistent CTA per SM, 16 warps (512 threads), two roles connected by mbarriers:
//
//   warps 8-11  producer of the CORE half, warps 12-15 producer of the GATE half of every 128-row tile (two
//               independent groups): 16 lanes x float4 per 64-float half-row (coalesced) gather + add the
//               first-layer rows, SiLU, store the [128 x 64] half-tile to shared memory (16-byte chunks
//               XOR-swizzled by row); BondConv also writes save_pre
//   warps 0-7   two consumer warpgroups, tile rows 0-63 / 64-127: each warp reads its A fragments from both
//               half-tiles (conflict-free), the warpgroup issues 8 k-steps x 3 split terms of wgmma m64n64k8
//               per half; the epilogue runs on the accumulator fragments (a row's 64 values sit in one lane
//               quad: LayerNorm by quad shuffles), SiLU (core) x sigmoid (gate) -> one [128 x 64] tile in
//               shared memory; then each of the 8 warps reduces a 16-row strip (x bond weights, read
//               coalesced) over runs of equal segment id: complete segments are stored, strip-boundary
//               partials go to `parts`
//
// A tiny second kernel (seg_stitch) adds the strip partials of every segment that spans strips, in strip
// order (deterministic, no atomics), and zeroes empty segments.
//
// Shared memory: 4 weight images (64 KB) + 2 half-tiles (64 KB) + the output tile (32 KB) + indices.
#include "gated_common.cuh"
#include "tc.cuh"

namespace chg {
namespace gated {
namespace {

constexpr int WS_THREADS = 512;  // 8 consumer warps (two warpgroups), 8 producer warps
constexpr int TR = 128;          // rows per tile
constexpr int HALF_BYTES = TR * 64 * 4;
constexpr int IMG_BYTES = 64 * 64 * 4;
constexpr int STRIP = 16;        // rows per reduction strip (one half-warp)

struct WsSmem {
  static constexpr int IMG_OFF = 0;                          // Bc_hi, Bc_lo, Bg_hi, Bg_lo
  static constexpr int HS_OFF = 4 * IMG_BYTES;               // 2 x [128][64] fp32, swizzled (core | gate producer)
  static constexpr int O_OFF = HS_OFF + 2 * HALF_BYTES;      // [128][64] fp32, swizzled: silu(core) * sigmoid(gate)
  static constexpr int GIDX_OFF = O_OFF + HALF_BYTES;        // 2 groups x 3 x 128 int
  static constexpr int EIDX_OFF = GIDX_OFF + 2 * 3 * TR * 4;  // 4 x 128 int: segment id, weight row, segment begin / end
  static constexpr int B2_OFF = EIDX_OFF + 4 * TR * 4;       // 128 floats
  static constexpr int LN_OFF = B2_OFF + 128 * 4;            // 256 floats
  static constexpr int TOTAL = LN_OFF + 256 * 4;
};

struct WsBars {
  uint64_t a_full[2], a_empty[2];
};

struct FusedArgs {
  const float* p_a;     // ATOM: pcn [N][256]        BOND: pij [Es][256]
  const float* p_b;     // ATOM: pe  [Eu][128]       BOND: px  [N][128]
  const float* p_c;     // BOND: pa [A][128], else null
  const float* wgt;     // ATOM: wag [Eu][64]        BOND: wbg_s [Es][64]
  const int32_t* idx0;  // row of p_a, first half = the SEGMENT id  (center | bond slot i)
  const int32_t* idx1;  // row of p_a, second half                  (nbr    | bond slot j)
  const int32_t* idx2;  // row of p_b                               (d2u    | atom)
  const int32_t* ptr;   // [n_seg + 1] CSR of idx0
  int32_t n_rows, n_seg;
  const float* w2t;     // [64][128]
  const float* b2;      // [128]
  const float* ln;      // [4][64] or null
  float* out;           // [n_seg][64]
  float* parts;         // [ceil(n_rows / 16)][2][64]
  float* save_pre;      // [rows][128] or null
  float* save_p;        // [rows][128] or null
};

// pull one 128-byte line towards L2 (no register, no dependency): the bond-weight rows of a tile, read after its products.
// The streamed rows (pa, saved pre / p, the per-bond products) are NOT prefetched a tile ahead: measured slower (DESIGN.md §4)
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// byte offset of 16-byte chunk c (0..15) of row r in a swizzled [128][64] fp32 tile
__device__ __forceinline__ int swz(int r, int c) { return r * 256 + ((c ^ (r & 7)) << 4); }

// image element (n, kk) = src[kk * ld + col0 + n]   (64 x 64, K-major, no swizzle), all threads of the CTA
__device__ __forceinline__ void build_image_ws(uint8_t* hi, uint8_t* lo, const float* __restrict__ src, int ld, int col0,
                                               int tid) {
  for (int i = tid; i < 4096; i += (int)blockDim.x) {
    const int kk = i >> 6, n = i & 63;
    uint32_t h, l;
    tc::split_tf32(__ldg(src + (size_t)kk * ld + col0 + n), h, l);
    const uint32_t off = tc::kmajor_offset(n, kk, 64);
    *reinterpret_cast<uint32_t*>(hi + off) = h;
    *reinterpret_cast<uint32_t*>(lo + off) = l;
  }
}

// ---- epilogue helpers on m64n64 accumulator fragments -----------------------------------------------------
// sum over the lane quad that holds one accumulator row
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}
// in place: d (+ b2) -> saved p (optional) -> LayerNorm (optional, per row over the quad; two-pass statistics)
__device__ __forceinline__ void bias_ln_frag(float (&d)[32], const float* s_b2, const float* s_gamma, const float* s_beta,
                                             bool use_ln, float* save_rows, int row0, int n_rows) {
#pragma unroll
  for (int i = 0; i < 32; ++i) d[i] += s_b2[tc::frag_col(i)];
  if (save_rows != nullptr) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int g = row0 + tc::frag_row(i);
      if (g < n_rows) *reinterpret_cast<float2*>(save_rows + (size_t)g * 128 + tc::frag_col(i)) = make_float2(d[i], d[i + 1]);
    }
  }
  if (!use_ln) return;
#pragma unroll
  for (int h = 0; h < 2; ++h) {  // h = 0: row frag_row(0), h = 1: row frag_row(0) + 8
    float s1 = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i)
      if (((i >> 1) & 1) == h) s1 += d[i];
    const float mean = quad_sum(s1) * (1.f / 64.f);
    float s2 = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i)
      if (((i >> 1) & 1) == h) s2 = fmaf(d[i] - mean, d[i] - mean, s2);
    const float rstd = 1.f / sqrtf(quad_sum(s2) * (1.f / 64.f) + LN_EPS);
#pragma unroll
    for (int i = 0; i < 32; ++i)
      if (((i >> 1) & 1) == h) d[i] = fmaf((d[i] - mean) * rstd, s_gamma[tc::frag_col(i)], s_beta[tc::frag_col(i)]);
  }
}

template <int MODE>
__global__ void __launch_bounds__(WS_THREADS, 1) gated_ws_fwd_kernel(const FusedArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* s_img = smem_raw + WsSmem::IMG_OFF;
  uint8_t* s_hs = smem_raw + WsSmem::HS_OFF;
  uint8_t* s_o = smem_raw + WsSmem::O_OFF;
  int* s_gidx = reinterpret_cast<int*>(smem_raw + WsSmem::GIDX_OFF);
  int* s_eidx = reinterpret_cast<int*>(smem_raw + WsSmem::EIDX_OFF);
  float* s_b2 = reinterpret_cast<float*>(smem_raw + WsSmem::B2_OFF);
  float* s_ln = reinterpret_cast<float*>(smem_raw + WsSmem::LN_OFF);
  __shared__ __align__(8) WsBars bars;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const bool use_ln = a.ln != nullptr;
  const int n_tiles = (a.n_rows + TR - 1) / TR;

  // ---- one-time setup: weight images, bias / LayerNorm rows, barriers ------------------------------------------
  build_image_ws(s_img, s_img + IMG_BYTES, a.w2t, 128, 0, tid);                     // core: (n=c, kk=k) = w2t[k][c]
  build_image_ws(s_img + 2 * IMG_BYTES, s_img + 3 * IMG_BYTES, a.w2t, 128, 64, tid);  // gate
  if (tid < 128) s_b2[tid] = a.b2[tid];
  if (tid < 256) s_ln[tid] = use_ln ? a.ln[tid] : 0.f;
  if (tid == 0) {
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&bars.a_full[i], 128);
      tc::mbar_init(&bars.a_empty[i], 256);
    }
    tc::mbar_fence_init();
  }
  tc::fence_async_smem();
  __syncthreads();

  if (warp >= 8) {
    // ============================ producer groups (gather -> SiLU -> half-tile) ============================
    const int half = (warp - 8) >> 2;            // 0: core columns, 1: gate columns
    const int gt = tid - 256 - half * 128;       // 0..127 inside the group
    const int tx = gt & 15, ty = gt >> 4;        // 16 lanes per row, 8 rows per pass
    int* gi = s_gidx + half * 3 * TR;
    uint8_t* stage = s_hs + half * HALF_BYTES;
    const int col = half * 64 + tx * 4;
    constexpr int PB = 4;  // rows gathered per batch (x 3-4 loads each in flight)
    int tl = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tl) {
      const int base = tile * TR;
      {
        const int r = min(base + gt, a.n_rows - 1);
        gi[gt] = a.idx0[r];
        gi[TR + gt] = a.idx1[r];
        gi[2 * TR + gt] = a.idx2[r];
      }
      tc::wg_barrier(1 + half, 128);  // indices visible
#pragma unroll 1
      for (int b = 0; b < 16 / PB; ++b) {
        float4 v[PB];
#pragma unroll
        for (int i = 0; i < PB; ++i) {
          const int row = ty + 8 * (b * PB + i);
          const float* s0 = a.p_a + (size_t)gi[row] * 256 + col;
          const float* s1 = a.p_a + (size_t)gi[TR + row] * 256 + 128 + col;
          const float* s2 = a.p_b + (size_t)gi[2 * TR + row] * 128 + col;
          v[i] = ldg4(s0) + ldg4(s1) + ldg4(s2);
          if (MODE == BOND) v[i] = v[i] + ldg4(a.p_c + (size_t)min(base + row, a.n_rows - 1) * 128 + col);
        }
        if (b == 0) tc::mbar_wait(&bars.a_empty[half], (tl & 1) ^ 1);  // the consumers have read the previous half-tile
#pragma unroll
        for (int i = 0; i < PB; ++i) {
          const int row = ty + 8 * (b * PB + i);
          if (a.save_pre != nullptr && base + row < a.n_rows) stg4(a.save_pre + (size_t)(base + row) * 128 + col, v[i]);
          *reinterpret_cast<float4*>(stage + swz(row, tx)) =
              make_float4(silu_f(v[i].x), silu_f(v[i].y), silu_f(v[i].z), silu_f(v[i].w));
        }
      }
      tc::wg_barrier(1 + half, 128);  // every thread of the group is done with the indices of this tile
      tc::mbar_arrive(&bars.a_full[half]);
    }
  } else {
    // ============================ consumers: warps 0-3 rows 0-63, warps 4-7 rows 64-127 ============================
    const int cw = warp >> 2;
    const int t = tid & 127;         // index-row duty: warps 0-3 segment rows, warps 4-7 weight rows
    const int row0 = cw * 64;
    int* s_seg = s_eidx;             // segment id of every tile row
    int* s_wrow = s_eidx + TR;       // row of the bond weight (ATOM: d2u; BOND: slot j - slot i is the segment id)
    int* s_sa = s_eidx + 2 * TR;     // ptr[seg], ptr[seg + 1] of every tile row
    int* s_sb = s_eidx + 3 * TR;
    const uint32_t img = tc::smem_u32(s_img);
    int tl = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tl) {
      const int base = tile * TR;
      {
        const int r = min(base + t, a.n_rows - 1);
        if (cw == 0) {
          const int seg = a.idx0[r];
          s_seg[t] = seg;
          s_sa[t] = __ldg(a.ptr + seg);
          s_sb[t] = __ldg(a.ptr + seg + 1);
        } else {
          const int wr = MODE == BOND ? a.idx1[r] : a.idx2[r];
          s_wrow[t] = wr;
          prefetch_l2(a.wgt + (size_t)wr * 64);  // the bond-weight row the strip reduction reads after the products
          prefetch_l2(a.wgt + (size_t)wr * 64 + 32);
        }
      }
      float dc[32], dg[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) dc[i] = dg[i] = 0.f;
      tc::mbar_wait(&bars.a_full[0], tl & 1);
      tc::wg_gemm_k64<64>(dc, [&](int r, int k) { return *reinterpret_cast<const float*>(s_hs + swz(row0 + r, k >> 2) + (k & 3) * 4); },
                          img, img + IMG_BYTES, 2048);
      tc::mbar_arrive(&bars.a_empty[0]);
      tc::mbar_wait(&bars.a_full[1], tl & 1);
      tc::wg_gemm_k64<64>(dg, [&](int r, int k) { return *reinterpret_cast<const float*>(s_hs + HALF_BYTES + swz(row0 + r, k >> 2) + (k & 3) * 4); },
                          img + 2 * IMG_BYTES, img + 3 * IMG_BYTES, 2048);
      tc::mbar_arrive(&bars.a_empty[1]);
      // epilogue: p = acc + b2 (saved), LayerNorm, silu(core) * sigmoid(gate) -> output tile
      float* save = a.save_p != nullptr ? a.save_p + (size_t)base * 128 : nullptr;
      bias_ln_frag(dc, s_b2, s_ln, s_ln + 64, use_ln, save, row0, a.n_rows - base);
      bias_ln_frag(dg, s_b2 + 64, s_ln + 128, s_ln + 192, use_ln, save != nullptr ? save + 64 : nullptr, row0, a.n_rows - base);
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int r = row0 + tc::frag_row(i), c = tc::frag_col(i);
        *reinterpret_cast<float2*>(s_o + swz(r, c >> 2) + (c & 3) * 4) =
            make_float2(silu_f(dc[i]) * sigmoid_f(dg[i]), silu_f(dc[i + 1]) * sigmoid_f(dg[i + 1]));
      }
      tc::wg_barrier(3, 256);

      // ---- segmented reduction: warp w owns the 16-row strip w, lane l the columns 2l, 2l+1 ----------------
      const int strip_lo = base + warp * STRIP;
      const int strip_hi = min(strip_lo + STRIP, a.n_rows);
      if (strip_lo < a.n_rows) {
        float2 w[STRIP];
#pragma unroll
        for (int i = 0; i < STRIP; ++i) {
          const int rr = warp * STRIP + i;
          const float2 w0 = __ldg(reinterpret_cast<const float2*>(a.wgt + (size_t)s_wrow[rr] * 64) + lane);
          if (MODE == ATOM) {
            w[i] = w0;
          } else {
            const float2 wi = __ldg(reinterpret_cast<const float2*>(a.wgt + (size_t)s_seg[rr] * 64) + lane);
            w[i] = make_float2(wi.x * w0.x, wi.y * w0.y);  // (o * w_i) * w_j
          }
        }
        float2 acc = make_float2(0.f, 0.f);
        int cur_row = warp * STRIP;  // first row of the current run
        auto emit = [&](int row0_, const float2& v) {
          const int seg = s_seg[row0_], sa = s_sa[row0_], sb = s_sb[row0_];
          float* dst;
          if (sa >= strip_lo && sb <= strip_hi) {
            dst = a.out + (size_t)seg * 64;  // the whole segment lies in this strip
          } else {
            dst = a.parts + ((size_t)(strip_lo / STRIP) * 2 + (sa < strip_lo ? 0 : 1)) * 64;
          }
          *reinterpret_cast<float2*>(dst + lane * 2) = v;
        };
#pragma unroll
        for (int i = 0; i < STRIP; ++i) {
          const int rr = warp * STRIP + i;
          if (strip_lo + i < strip_hi) {
            if (s_seg[rr] != s_seg[cur_row]) {
              emit(cur_row, acc);
              cur_row = rr;
              acc = make_float2(0.f, 0.f);
            }
            const float2 o = *reinterpret_cast<const float2*>(s_o + swz(rr, lane >> 1) + (lane & 1) * 8);
            acc.x = fmaf(o.x, w[i].x, acc.x);
            acc.y = fmaf(o.y, w[i].y, acc.y);
          }
        }
        emit(cur_row, acc);
      }
      tc::wg_barrier(3, 256);  // the output tile and the index rows are free for the next tile
    }
  }
}

// out[s] for every segment that spans more than one strip (sum of its strip partials, in strip order) and for
// every empty segment (zeros); segments inside one strip were stored by the main kernel.
__global__ void seg_stitch_kernel(const int32_t* __restrict__ ptr, int n_seg, const float* __restrict__ parts,
                                  float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int s = idx >> 4, l = idx & 15;
  if (s >= n_seg) return;
  const int a = ptr[s], b = ptr[s + 1];
  if (a >= b) {
    stg4(out + (size_t)s * 64 + l * 4, make_float4(0.f, 0.f, 0.f, 0.f));
    return;
  }
  const int k0 = a / STRIP, k1 = (b - 1) / STRIP;
  if (k0 == k1) return;
  float4 acc = ldg4(parts + ((size_t)k0 * 2 + 1) * 64 + l * 4);
  for (int k = k0 + 1; k <= k1; ++k) acc = acc + ldg4(parts + ((size_t)k * 2) * 64 + l * 4);
  stg4(out + (size_t)s * 64 + l * 4, acc);
}

template <int MODE>
int launch_fused(const FusedArgs& a, cudaStream_t stream) {
  if (a.n_seg == 0) return CHG_OK;
  if (a.n_rows > 0) {
    static bool attr_set[MAX_DEVICES] = {};  // per device: the attribute belongs to its context
    bool& set = attr_set[device_ordinal()];
    if (!set) {
      CHG_CUDA(cudaFuncSetAttribute(gated_ws_fwd_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, WsSmem::TOTAL));
      set = true;
    }
    const int n_tiles = (a.n_rows + TR - 1) / TR;
    gated_ws_fwd_kernel<MODE><<<min(n_tiles, sm_count()), WS_THREADS, WsSmem::TOTAL, stream>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      set_error("gated_ws_fwd_kernel: launch failed: %s", cudaGetErrorString(e));
      return CHG_ERR_CUDA;
    }
    count_launch();
  }
  seg_stitch_kernel<<<(a.n_seg * 16 + 255) / 256, 256, 0, stream>>>(a.ptr, a.n_seg, a.parts, a.out);
  CHG_LAUNCH_END();
}

}  // namespace

int atom_conv_fused_ws(const float* pcn, const float* pe, const float* wag, const int32_t* center, const int32_t* nbr,
                       const int32_t* d2u, const int32_t* ptr_c, int n_edges, int n_atoms, const float* w2t, const float* b2,
                       const float* ln, float* agg, float* save_p, float* parts, cudaStream_t stream) {
  FusedArgs a{pcn, pe, nullptr, wag, center, nbr, d2u, ptr_c, n_edges, n_atoms, w2t, b2, ln, agg, parts, nullptr, save_p};
  return launch_fused<ATOM>(a, stream);
}

int bond_conv_fused_ws(const float* pij, const float* px, const float* pa, const float* wbg, const int32_t* ang_atom,
                       const int32_t* ang_i, const int32_t* ang_j, const int32_t* ptr_i, int n_angles, int n_slots,
                       const float* w2t, const float* b2, const float* ln, float* agg, float* save_pre, float* save_p,
                       float* parts, cudaStream_t stream) {
  FusedArgs a{pij, px, pa, wbg, ang_i, ang_j, ang_atom, ptr_i, n_angles, n_slots, w2t, b2, ln, agg, parts, save_pre, save_p};
  return launch_fused<BOND>(a, stream);
}

}  // namespace gated
}  // namespace chg

using namespace chg;

// ---- C ABI: fused message + aggregation (include/chgnet_b200.h) -------------------------------------------------
extern "C" int64_t chg_gated_fused_workspace_floats(int32_t n_rows) {
  if (n_rows < 0) return -1;
  const int64_t msg = (int64_t)n_rows * 64, parts = ((int64_t)n_rows + 15) / 16 * 128;
  return (msg > parts ? msg : parts) + 64;
}

extern "C" int chg_atom_conv_fused(const float* pcn, const float* pe, const float* wag, const int32_t* center,
                                   const int32_t* nbr, const int32_t* d2u, const int32_t* ptr_c, int32_t n_edges,
                                   int32_t n_atoms, const float* w2t, const float* b2, const float* ln, float* agg,
                                   float* save_p, float* work, void* stream) {
  CHG_CHECK_ARG(n_edges >= 0 && n_atoms >= 0, "negative size");
  if (n_atoms == 0) return CHG_OK;
  CHG_CHECK_ARG(ptr_c && agg, "null pointer");
  CHG_CHECK_ARG(n_edges == 0 || (pcn && pe && wag && center && nbr && d2u && w2t && b2 && work), "null pointer");
  // tiny inputs (a few tiles) are launch-bound: the persistent tensor-core kernel's fixed cost (weight images) loses there
  if (gated_impl() == 3 && n_edges >= ws_min_rows())
    return gated::atom_conv_fused_ws(pcn, pe, wag, center, nbr, d2u, ptr_c, n_edges, n_atoms, w2t, b2, ln, agg, save_p, work,
                                     as_stream(stream));
  // A/B implementations 0..2: the unfused pair (message kernel -> segmented sum), the message in `work`
  const int rc = chg_atom_conv_fwd(pcn, pe, wag, center, nbr, d2u, n_edges, w2t, b2, ln, work, save_p, nullptr, stream);
  if (rc != CHG_OK) return rc;
  return chg_segment_sum(work, 64, nullptr, ptr_c, n_atoms, n_edges, 0, agg, 64, stream);
}

extern "C" int chg_bond_conv_fused(const float* pij, const float* px, const float* pa, const float* wbg,
                                   const int32_t* ang_atom, const int32_t* ang_i, const int32_t* ang_j,
                                   const int32_t* ptr_i, int32_t n_angles, int32_t n_slots, const float* w2t,
                                   const float* b2, const float* ln, float* agg, float* save_pre, float* save_p,
                                   float* work, void* stream) {
  CHG_CHECK_ARG(n_angles >= 0 && n_slots >= 0, "negative size");
  if (n_slots == 0) return CHG_OK;
  CHG_CHECK_ARG(ptr_i && agg, "null pointer");
  CHG_CHECK_ARG(n_angles == 0 || (pij && px && pa && wbg && ang_atom && ang_i && ang_j && w2t && b2 && work), "null pointer");
  if (gated_impl() == 3 && n_angles >= ws_min_rows())
    return gated::bond_conv_fused_ws(pij, px, pa, wbg, ang_atom, ang_i, ang_j, ptr_i, n_angles, n_slots, w2t, b2, ln, agg,
                                     save_pre, save_p, work, as_stream(stream));
  const int rc = chg_bond_conv_fwd(pij, px, pa, wbg, ang_atom, ang_i, ang_j, n_angles, w2t, b2, ln, work, save_pre, save_p, stream);
  if (rc != CHG_OK) return rc;
  return chg_segment_sum(work, 64, nullptr, ptr_i, n_slots, n_angles, 0, agg, 64, stream);
}

// =====================================================================================================================
// Reverse of the AtomConv / BondConv message (same entry points and arithmetic as gated_bwd_kernel<MODE, false> in
// gated.cu; reference: autograd of layers.py:113-121, 238-249): warp-specialised wgmma version.
//
//   warps 0-7   P  16 lanes x float4 per 64-wide half-row: saved p -> LayerNorm statistics (shuffles) -> gates,
//                  bond-weight gradients (stored), LayerNorm reverse -> g_p tile in shared memory (two swizzled
//                  halves)
//   warps 8-15  F  two warpgroups, tile rows 0-63 / 64-127: g_h = g_p . W2 per half (A fragments read from the g_p
//                  tile, 8 k-steps x 3 split terms of wgmma m64n64k8), accumulator fragments -> g_h tile in shared
//                  memory; group barrier; then 16 lanes x float4 per half-row: g_pre = g_h * silu'(pre), pre
//                  recomputed from the first-layer rows (AtomConv) or read from save_pre (BondConv), coalesced stores
// =====================================================================================================================
namespace chg {
namespace gated {
namespace {

struct WsBwdSmem {
  static constexpr int IMG_OFF = 0;                         // W2 images: core hi, lo, gate hi, lo
  static constexpr int T1_OFF = 4 * IMG_BYTES;              // g_p tile: 2 x [128][64] fp32 swizzled
  static constexpr int T2_OFF = T1_OFF + 2 * HALF_BYTES;    // g_h tile: 2 x [128][64] fp32 swizzled
  static constexpr int PIDX_OFF = T2_OFF + 2 * HALF_BYTES;  // 3 x 128 int (P group)
  static constexpr int FIDX_OFF = PIDX_OFF + 3 * TR * 4;    // 3 x 128 int (F group)
  static constexpr int LN_OFF = FIDX_OFF + 3 * TR * 4;      // 256 floats
  static constexpr int TOTAL = LN_OFF + 256 * 4;
};

struct WsBwdBars {
  uint64_t a_full, a_empty;
};

template <int MODE>
__global__ void __launch_bounds__(WS_THREADS, 1) gated_ws_bwd_kernel(const BwdArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* s_img = smem_raw + WsBwdSmem::IMG_OFF;
  uint8_t* s_t1 = smem_raw + WsBwdSmem::T1_OFF;
  uint8_t* s_t2 = smem_raw + WsBwdSmem::T2_OFF;
  int* s_pidx = reinterpret_cast<int*>(smem_raw + WsBwdSmem::PIDX_OFF);
  int* s_fidx = reinterpret_cast<int*>(smem_raw + WsBwdSmem::FIDX_OFF);
  float* s_ln = reinterpret_cast<float*>(smem_raw + WsBwdSmem::LN_OFF);
  __shared__ __align__(8) WsBwdBars bars;

  const int tid = threadIdx.x, warp = tid >> 5;
  const bool use_ln = a.ln != nullptr;
  const int n_tiles = (a.n_rows + TR - 1) / TR;

  // g_h[k] = sum_c g_p[c] W2[c][k]: image element (n = k, kk = c) = w2[c][k]
  build_image_ws(s_img, s_img + IMG_BYTES, a.w2, 64, 0, tid);
  build_image_ws(s_img + 2 * IMG_BYTES, s_img + 3 * IMG_BYTES, a.w2 + 64 * 64, 64, 0, tid);
  if (tid < 256) s_ln[tid] = use_ln ? a.ln[tid] : 0.f;
  if (tid == 0) {
    tc::mbar_init(&bars.a_full, 256);
    tc::mbar_init(&bars.a_empty, 256);
    tc::mbar_fence_init();
  }
  tc::fence_async_smem();
  __syncthreads();

  if (warp < 8) {
    // ============================ P: saved p -> g_p -> A operand ============================
    const int t = tid;                   // 0..255
    const int tx = t & 15, ty = t >> 4;  // 16 lanes per row, 16 rows per pass
    const int c0 = tx * 4;
    int tl = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tl) {
      const int base = tile * TR;
      if (t < TR) {
        const int r = min(base + t, a.n_rows - 1);
        s_pidx[t] = a.idx0[r];
        s_pidx[TR + t] = a.idx1[r];
        if (MODE == ATOM) s_pidx[2 * TR + t] = a.idx2[r];
      }
      tc::wg_barrier(1, 256);  // indices visible
      float4 g1, g2, b1, b2v;
      if (use_ln) {
        g1 = lds4(s_ln + c0);
        b1 = lds4(s_ln + 64 + c0);
        g2 = lds4(s_ln + 128 + c0);
        b2v = lds4(s_ln + 192 + c0);
      }
      tc::mbar_wait(&bars.a_empty, (tl & 1) ^ 1);  // the MMAs of the previous tile have read the g_p tile
#pragma unroll 2
      for (int pass = 0; pass < 8; ++pass) {
        const int row = pass * 16 + ty;
        const int g = base + row;
        const bool valid = g < a.n_rows;
        const int r = min(g, a.n_rows - 1);
        const float4 pc4 = ldg4(a.save_p + (size_t)r * 128 + c0);
        const float4 pg4 = ldg4(a.save_p + (size_t)r * 128 + 64 + c0);
        float4 gm, wv;
        if (MODE == ATOM) {
          gm = ldg4(a.g_in + (size_t)s_pidx[row] * 64 + c0);
          wv = ldg4(a.wgt + (size_t)s_pidx[2 * TR + row] * 64 + c0);
        } else {
          gm = ldg4(a.g_in + (size_t)s_pidx[row] * 64 + c0);
          wv = ldg4(a.wgt + (size_t)s_pidx[row] * 64 + c0);
        }
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
          if (valid) stg4(a.g_w0 + (size_t)g * 64 + c0, gm * o);
          go = gm * wv;
        } else {
          const float4 wj = ldg4(a.wgt + (size_t)s_pidx[TR + row] * 64 + c0);
          const float4 gmo = gm * o;
          if (valid) {
            stg4(a.g_w0 + (size_t)g * 64 + c0, gmo * wj);
            stg4(a.g_w1 + (size_t)g * 64 + c0, gmo * wv);
          }
          go = gm * wv * wj;
        }
        float gy1[4], gy2[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float gj = f4at(go, j);
          gy1[j] = gj * gate[j] * (s1[j] * fmaf(y1[j], 1.f - s1[j], 1.f));
          gy2[j] = gj * core[j] * gate[j] * (1.f - gate[j]);
        }
        if (use_ln) {
          // g_p = rstd * (gx - mean(gx) - xhat * mean(gx * xhat)), gx = gy * gamma
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
        *reinterpret_cast<float4*>(s_t1 + swz(row, tx)) = make_float4(gy1[0], gy1[1], gy1[2], gy1[3]);
        *reinterpret_cast<float4*>(s_t1 + HALF_BYTES + swz(row, tx)) = make_float4(gy2[0], gy2[1], gy2[2], gy2[3]);
      }
      tc::wg_barrier(1, 256);  // every thread is done with the indices of this tile
      tc::mbar_arrive(&bars.a_full);
    }
  } else {
    // ============================ F: g_h = g_p . W2, then g_pre = g_h * silu'(pre) ============================
    const int t = tid - 256;             // 0..255
    const int tx = t & 15, ty = t >> 4;
    const int c0 = tx * 4;
    const int row0 = ((warp - 8) >> 2) * 64;  // this warpgroup's rows of the products
    const uint32_t img = tc::smem_u32(s_img);
    int tl = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tl) {
      const int base = tile * TR;
      if (MODE == ATOM && t < TR) {
        const int r = min(base + t, a.n_rows - 1);
        s_fidx[t] = a.idx0[r];
        s_fidx[TR + t] = a.idx1[r];
        s_fidx[2 * TR + t] = a.idx2[r];
      }
      tc::mbar_wait(&bars.a_full, tl & 1);
#pragma unroll 1
      for (int half = 0; half < 2; ++half) {
        float d[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) d[i] = 0.f;
        const uint8_t* src = s_t1 + half * HALF_BYTES;
        tc::wg_gemm_k64<64>(d, [&](int r, int k) { return *reinterpret_cast<const float*>(src + swz(row0 + r, k >> 2) + (k & 3) * 4); },
                            img + half * 2 * IMG_BYTES, img + (half * 2 + 1) * IMG_BYTES, 2048);
        uint8_t* dst = s_t2 + half * HALF_BYTES;
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int r = row0 + tc::frag_row(i), c = tc::frag_col(i);
          *reinterpret_cast<float2*>(dst + swz(r, c >> 2) + (c & 3) * 4) = make_float2(d[i], d[i + 1]);
        }
      }
      tc::mbar_arrive(&bars.a_empty);
      tc::wg_barrier(2, 256);  // the g_h tile (and the index rows) are complete
#pragma unroll 2
      for (int pass = 0; pass < 8; ++pass) {
        const int row = pass * 16 + ty;
        const int g = base + row;
        float4 vc, vg;
        if (MODE == ATOM) {
          const float* s0 = a.p_a + (size_t)s_fidx[row] * 256 + c0;
          const float* s1 = a.p_a + (size_t)s_fidx[TR + row] * 256 + 128 + c0;
          const float* s2 = a.p_b + (size_t)s_fidx[2 * TR + row] * 128 + c0;
          vc = ldg4(s0) + ldg4(s1) + ldg4(s2);
          vg = ldg4(s0 + 64) + ldg4(s1 + 64) + ldg4(s2 + 64);
        } else {
          const int r = min(g, a.n_rows - 1);
          vc = ldg4(a.save_pre + (size_t)r * 128 + c0);
          vg = ldg4(a.save_pre + (size_t)r * 128 + 64 + c0);
        }
        const float4 hc = *reinterpret_cast<const float4*>(s_t2 + swz(row, tx));
        const float4 hg = *reinterpret_cast<const float4*>(s_t2 + HALF_BYTES + swz(row, tx));
        if (g < a.n_rows) {
          stg4(a.g_pre + (size_t)g * 128 + c0,
               make_float4(hc.x * dsilu_f(vc.x), hc.y * dsilu_f(vc.y), hc.z * dsilu_f(vc.z), hc.w * dsilu_f(vc.w)));
          stg4(a.g_pre + (size_t)g * 128 + 64 + c0,
               make_float4(hg.x * dsilu_f(vg.x), hg.y * dsilu_f(vg.y), hg.z * dsilu_f(vg.z), hg.w * dsilu_f(vg.w)));
        }
      }
      tc::wg_barrier(2, 256);  // the g_h tile can be overwritten
    }
  }
}

template <int MODE>
int launch_ws_bwd(const BwdArgs& a, cudaStream_t stream) {
  if (a.n_rows == 0) return CHG_OK;
  static bool attr_set[MAX_DEVICES] = {};  // per device: the attribute belongs to its context
  bool& set = attr_set[device_ordinal()];
  if (!set) {
    CHG_CUDA(cudaFuncSetAttribute(gated_ws_bwd_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, WsBwdSmem::TOTAL));
    set = true;
  }
  const int n_tiles = (a.n_rows + TR - 1) / TR;
  gated_ws_bwd_kernel<MODE><<<min(n_tiles, sm_count()), WS_THREADS, WsBwdSmem::TOTAL, stream>>>(a);
  CHG_LAUNCH_END();
}

}  // namespace

int atom_conv_bwd_ws(const BwdArgs& a, cudaStream_t stream) { return launch_ws_bwd<ATOM>(a, stream); }
int bond_conv_bwd_ws(const BwdArgs& a, cudaStream_t stream) { return launch_ws_bwd<BOND>(a, stream); }

}  // namespace gated
}  // namespace chg
