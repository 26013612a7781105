// Second-order gated-MLP kernels: the TANGENT of AtomConv / BondConv / AngleUpdate along a fixed
// direction of the edge vectors, and the reverse of (primal, tangent) — what a loss on forces /
// stresses adds to a training step (reference model.py:518-535 create_graph=True, trainer.py:409).
//
// Per row (edge / angle), with the first-order kernels' notation (gated.cu):
//   pre -> h = silu(pre) -> p = W2 h + b2 -> y = LN(p) -> o = silu(y_core) sigmoid(y_gate) -> out = o w
//   tangent:  pre' given;  p' = W2 (silu'(pre) pre');  y' = LN'(p)[p'];  o' ;  out' = o' w + o w'
//   reverse of the scalar  S = <bar, out> + <lam, out'>   (bar = adjoint of out from the second reverse
//   pass, lam = dE/d out from the force pass; pre', w' held fixed):
//       u      = dS/dp      = LN/act reverse of (bar w + lam w') + Hessian term of <lam w, o'>
//       bar_pre= silu'(pre) W2^T u + silu''(pre) pre' W2^T g_p_lam        (g_p_lam = dE/dp, force pass)
//       bar_w  = bar o + lam o'
// oracle/kernel_specs.py (_gate_tan, _gate_bwd2) states the same maths in torch; the CPU tests check
// the whole chain against autograd's double backward.
//
// Thread map as in gated.cu: 256 threads = 16 (ty) x 16 (tx); a thread owns rows ty*4..+3 and columns
// tx*4..+3 of both halves; LayerNorm reductions run over the 16 tx lanes.
#include "gated_common.cuh"

namespace chg {
namespace {

using namespace gated;

struct TanArgs {
  const float* pa_d;    // tangent of p_a  (ATOM: pcn' [N][256]; BOND/ANGLE: pij' [Es][256])
  const float* pb_d;    // tangent of p_b  (ATOM: pe' [Eu][128]; BOND/ANGLE: px' [N][128])
  const float* pc_d;    // BOND/ANGLE: pa' [A][128]
  const float* feat_d;  // ANGLE: tangent of the angle features [A][64]
  const float* wgt;     // ATOM: wag; BOND: wbg (compact)
  const float* wgt_d;   // their tangents
  const int32_t* idx0;
  const int32_t* idx1;
  const int32_t* idx2;
  int32_t n_rows;
  const float* save_pre;  // ATOM / BOND
  const float* save_p;
  const float* w2t;  // [64][128]
  const float* ln;
  float* out_d;  // [rows][64]
  float* pre_d;  // [rows][128] (ATOM / BOND)
  float* p_d;    // [rows][128]
};

struct Bwd2Args {
  const float* save_pre;
  const float* save_p;
  const float* pre_d;
  const float* p_d;
  const float* g_p_lam;  // ATOM / BOND: dE/dp of the force pass [rows][128]
  const float* wgt;
  const float* wgt_d;
  const int32_t* idx_seed;  // row of lam_in / bar_in (ATOM: center; BOND: bond i); ANGLE: the row itself
  const int32_t* idx_w0;    // ATOM: d2u; BOND: bond i
  const int32_t* idx_w1;    // BOND: bond j
  int32_t n_rows;
  const float* lam_in;  // may be null (ANGLE) = 0
  const float* bar_in;  // may be null (ANGLE) = 0
  const float* w2;      // [128][64]
  const float* ln;
  float* bar_pre;  // [rows][128]
  float* bar_w0;   // ATOM: bar_w; BOND: bar_wi
  float* bar_w1;   // BOND: bar_wj
  float* u_out;    // [rows][128] (ATOM / BOND)
  double* g_ln;    // [4][64] accumulated, or null
};

__device__ __forceinline__ float d2silu_f(float x) {
  const float s = sigmoid_f(x);
  return s * (1.f - s) * fmaf(x, 1.f - 2.f * s, 2.f);
}

// one branch (core or gate) of one row, 4 of its 64 columns in this thread
struct Branch {
  float y[4], yd[4], xh[4], xd[4], pd[4];
  float rstd, m2;  // m2 = mean(xhat * pd)
};

__device__ __forceinline__ void branch_tan(Branch& br, const float (&p)[4], const float (&pd)[4], bool use_ln,
                                           const float4& gamma, const float4& beta) {
#pragma unroll
  for (int j = 0; j < 4; ++j) br.pd[j] = pd[j];
  if (!use_ln) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      br.y[j] = p[j];
      br.yd[j] = pd[j];
      br.xh[j] = br.xd[j] = 0.f;
    }
    br.rstd = 1.f;
    br.m2 = 0.f;
    return;
  }
  ln_stats(p, br.xh, br.rstd);
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    s1 += pd[j];
    s2 = fmaf(br.xh[j], pd[j], s2);
  }
  const float m1 = sum16(s1) * (1.f / 64.f);
  br.m2 = sum16(s2) * (1.f / 64.f);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    br.xd[j] = br.rstd * (pd[j] - m1 - br.xh[j] * br.m2);
    br.y[j] = fmaf(br.xh[j], f4at(gamma, j), f4at(beta, j));
    br.yd[j] = f4at(gamma, j) * br.xd[j];
  }
}

// q = d/dp of [ <gy, y(p)> + <kap, ydot(p, pd)> ] for one branch; also the LayerNorm affine gradients
__device__ __forceinline__ void branch_bwd2(const Branch& br, const float (&gy)[4], const float (&kap)[4], bool use_ln,
                                            const float4& gamma, float (&q)[4], float* acc_gamma, float* acc_beta,
                                            bool valid) {
  if (!use_ln) {
#pragma unroll
    for (int j = 0; j < 4; ++j) q[j] = gy[j];
    return;
  }
  if (valid) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      acc_gamma[j] += fmaf(gy[j], br.xh[j], kap[j] * br.xd[j]);
      acc_beta[j] += gy[j];
    }
  }
  float kk[4], s_kx = 0.f, s_kxd = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    kk[j] = kap[j] * f4at(gamma, j);
    s_kx = fmaf(kk[j], br.xh[j], s_kx);
    s_kxd = fmaf(kk[j], br.xd[j], s_kxd);
  }
  s_kx = sum16(s_kx);
  s_kxd = sum16(s_kxd);
  float v[4], sv = 0.f, svx = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    v[j] = fmaf(gy[j], f4at(gamma, j), br.rstd * (-kk[j] * br.m2 - s_kx * br.pd[j] * (1.f / 64.f)));
    sv += v[j];
    svx = fmaf(v[j], br.xh[j], svx);
  }
  sv = sum16(sv) * (1.f / 64.f);
  svx = sum16(svx) * (1.f / 64.f);
#pragma unroll
  for (int j = 0; j < 4; ++j)
    q[j] = br.rstd * (v[j] - sv - br.xh[j] * svx) - br.rstd * br.xh[j] * s_kxd * (1.f / 64.f);
}

__device__ __forceinline__ void load8(const float* base, size_t row, int c0, float (&c)[4], float (&g)[4]) {
  const float4 vc = ldg4(base + row * 128 + c0), vg = ldg4(base + row * 128 + 64 + c0);
  c[0] = vc.x; c[1] = vc.y; c[2] = vc.z; c[3] = vc.w;
  g[0] = vg.x; g[1] = vg.y; g[2] = vg.z; g[3] = vg.w;
}

template <int MODE>
struct TanSmem {
  static constexpr bool HAS_W2 = MODE != ANGLE;
  static constexpr int W2_OFF = 0;
  static constexpr int TILE_OFF = W2_OFF + (HAS_W2 ? 64 * 128 : 0);
  static constexpr int LN_OFF = TILE_OFF + (HAS_W2 ? TM * HS : 0);
  static constexpr int IDX_OFF = LN_OFF + 256;
  static constexpr int TOTAL_BYTES = (IDX_OFF + 3 * TM) * 4;
};

template <int MODE>
__global__ void __launch_bounds__(NTHR, 2) gated_tan_kernel(const TanArgs a) {
  using L = TanSmem<MODE>;
  extern __shared__ __align__(16) float smem[];
  float* s_w2t = smem + L::W2_OFF;
  float* s_tile = smem + L::TILE_OFF;
  float* s_ln = smem + L::LN_OFF;
  int* s_idx = reinterpret_cast<int*>(smem + L::IDX_OFF);
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int r0 = ty * 4, c0 = tx * 4;
  const bool use_ln = a.ln != nullptr;
  if (L::HAS_W2) copy_to_smem(s_w2t, a.w2t, 64 * 128, tid);
  if (use_ln) s_ln[tid] = a.ln[tid];

  const int n_tiles = (a.n_rows + TM - 1) / TM;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int base = tile * TM;
    __syncthreads();
    if (tid < TM) {
      const int r = min(base + tid, a.n_rows - 1);
      s_idx[tid] = a.idx0[r];
      s_idx[TM + tid] = a.idx1[r];
      s_idx[2 * TM + tid] = a.idx2[r];
    }
    __syncthreads();
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    gather_pre<TM>(acc, a.pa_d, a.pb_d, a.pc_d, s_idx, base, a.n_rows, r0, c0);  // pre'
    if (L::HAS_W2) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int g = base + r0 + i;
        const size_t r = (size_t)min(g, a.n_rows - 1);
        if (g < a.n_rows) {
          stg4(a.pre_d + (size_t)g * 128 + c0, make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]));
          stg4(a.pre_d + (size_t)g * 128 + 64 + c0, make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]));
        }
        float pc[4], pg[4];
        load8(a.save_pre, r, c0, pc, pg);
        sts4(s_tile + (r0 + i) * HS + c0, make_float4(dsilu_f(pc[0]) * acc[i][0], dsilu_f(pc[1]) * acc[i][1],
                                                     dsilu_f(pc[2]) * acc[i][2], dsilu_f(pc[3]) * acc[i][3]));
        sts4(s_tile + (r0 + i) * HS + 64 + c0, make_float4(dsilu_f(pg[0]) * acc[i][4], dsilu_f(pg[1]) * acc[i][5],
                                                          dsilu_f(pg[2]) * acc[i][6], dsilu_f(pg[3]) * acc[i][7]));
      }
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
      gemm_blockdiag(acc, s_tile, s_w2t, s_w2t + 64, 128, r0, c0);  // p' = W2 h'
    }
    float4 g1 = make_float4(1.f, 1.f, 1.f, 1.f), b1 = make_float4(0.f, 0.f, 0.f, 0.f), g2 = g1, b2v = b1;
    if (use_ln) {
      g1 = lds4(s_ln + c0);
      b1 = lds4(s_ln + 64 + c0);
      g2 = lds4(s_ln + 128 + c0);
      b2v = lds4(s_ln + 192 + c0);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = r0 + i;
      const int g = base + row;
      const bool valid = g < a.n_rows;
      const size_t r = (size_t)min(g, a.n_rows - 1);
      if (valid) {
        stg4(a.p_d + (size_t)g * 128 + c0, make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]));
        stg4(a.p_d + (size_t)g * 128 + 64 + c0, make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]));
      }
      float pc[4], pg[4];
      load8(a.save_p, r, c0, pc, pg);
      const float pdc[4] = {acc[i][0], acc[i][1], acc[i][2], acc[i][3]};
      const float pdg[4] = {acc[i][4], acc[i][5], acc[i][6], acc[i][7]};
      Branch bc, bg;
      branch_tan(bc, pc, pdc, use_ln, g1, b1);
      branch_tan(bg, pg, pdg, use_ln, g2, b2v);
      float4 o, od;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float s1 = sigmoid_f(bc.y[j]), t = sigmoid_f(bg.y[j]);
        const float core = bc.y[j] * s1, dcore = s1 * fmaf(bc.y[j], 1.f - s1, 1.f);
        f4at(o, j) = core * t;
        f4at(od, j) = dcore * t * bc.yd[j] + core * t * (1.f - t) * bg.yd[j];
      }
      float4 res;
      if (MODE == ATOM) {
        const size_t u = (size_t)s_idx[2 * TM + row];
        res = od * ldg4(a.wgt + u * 64 + c0) + o * ldg4(a.wgt_d + u * 64 + c0);
      } else if (MODE == BOND) {
        const size_t bi = (size_t)s_idx[row], bj = (size_t)s_idx[TM + row];
        const float4 wi = ldg4(a.wgt + bi * 64 + c0), wj = ldg4(a.wgt + bj * 64 + c0);
        const float4 wdi = ldg4(a.wgt_d + bi * 64 + c0), wdj = ldg4(a.wgt_d + bj * 64 + c0);
        res = od * wi * wj + o * (wdi * wj + wi * wdj);
      } else {
        res = od + ldg4(a.feat_d + r * 64 + c0);
      }
      if (valid) stg4(a.out_d + (size_t)g * 64 + c0, res);
    }
  }
}

template <int MODE>
struct Bwd2Smem {
  static constexpr bool HAS_W2 = MODE != ANGLE;
  static constexpr int W2_OFF = 0;
  static constexpr int TILE_OFF = W2_OFF + (HAS_W2 ? 128 * 64 : 0);
  static constexpr int LN_OFF = TILE_OFF + (HAS_W2 ? TM * HS : 0);
  static constexpr int IDX_OFF = LN_OFF + 256;
  static constexpr int BODY_BYTES = (IDX_OFF + 3 * TM) * 4;
  static constexpr int TOTAL_BYTES = BODY_BYTES > 16 * 256 * 4 ? BODY_BYTES : 16 * 256 * 4;
};

template <int MODE>
__global__ void __launch_bounds__(NTHR, 2) gated_bwd2_kernel(const Bwd2Args a) {
  using L = Bwd2Smem<MODE>;
  extern __shared__ __align__(16) float smem[];
  float* s_w2 = smem + L::W2_OFF;   // [128][64]
  float* s_g = smem + L::TILE_OFF;  // [64][HS]
  float* s_ln = smem + L::LN_OFF;
  int* s_idx = reinterpret_cast<int*>(smem + L::IDX_OFF);
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int r0 = ty * 4, c0 = tx * 4;
  const bool use_ln = a.ln != nullptr;
  if (L::HAS_W2) copy_to_smem(s_w2, a.w2, 128 * 64, tid);
  if (use_ln) s_ln[tid] = a.ln[tid];
  float ln_acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) ln_acc[j] = 0.f;

  const int n_tiles = (a.n_rows + TM - 1) / TM;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int base = tile * TM;
    __syncthreads();
    if (MODE != ANGLE && tid < TM) {
      const int r = min(base + tid, a.n_rows - 1);
      s_idx[tid] = a.idx_seed[r];
      s_idx[TM + tid] = a.idx_w0[r];
      if (MODE == BOND) s_idx[2 * TM + tid] = a.idx_w1[r];
    }
    __syncthreads();
    float4 g1 = make_float4(1.f, 1.f, 1.f, 1.f), b1 = make_float4(0.f, 0.f, 0.f, 0.f), g2 = g1, b2v = b1;
    if (use_ln) {
      g1 = lds4(s_ln + c0);
      b1 = lds4(s_ln + 64 + c0);
      g2 = lds4(s_ln + 128 + c0);
      b2v = lds4(s_ln + 192 + c0);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = r0 + i;
      const int g = base + row;
      const bool valid = g < a.n_rows;
      const size_t r = (size_t)min(g, a.n_rows - 1);
      float pc[4], pg[4], pdc[4], pdg[4];
      load8(a.save_p, r, c0, pc, pg);
      load8(a.p_d, r, c0, pdc, pdg);
      Branch bc, bg;
      branch_tan(bc, pc, pdc, use_ln, g1, b1);
      branch_tan(bg, pg, pdg, use_ln, g2, b2v);
      // seeds: bar (adjoint of out in this pass), lam (dE/d out of the force pass)
      float4 lam = make_float4(0.f, 0.f, 0.f, 0.f), bar = lam;
      if (MODE == ANGLE) {
        if (a.lam_in != nullptr) lam = ldg4(a.lam_in + r * 64 + c0);
        if (a.bar_in != nullptr) bar = ldg4(a.bar_in + r * 64 + c0);
      } else {
        lam = ldg4(a.lam_in + (size_t)s_idx[row] * 64 + c0);
        bar = ldg4(a.bar_in + (size_t)s_idx[row] * 64 + c0);
      }
      float4 go, aa;  // effective seed on o, and the weight of o' in S
      float4 o, od;
      float s1[4], t[4], core[4], dcore[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s1[j] = sigmoid_f(bc.y[j]);
        t[j] = sigmoid_f(bg.y[j]);
        core[j] = bc.y[j] * s1[j];
        dcore[j] = s1[j] * fmaf(bc.y[j], 1.f - s1[j], 1.f);
        f4at(o, j) = core[j] * t[j];
        f4at(od, j) = dcore[j] * t[j] * bc.yd[j] + core[j] * t[j] * (1.f - t[j]) * bg.yd[j];
      }
      if (MODE == ATOM) {
        const size_t u = (size_t)s_idx[TM + row];
        const float4 w = ldg4(a.wgt + u * 64 + c0), wd = ldg4(a.wgt_d + u * 64 + c0);
        if (valid) stg4(a.bar_w0 + (size_t)g * 64 + c0, bar * o + lam * od);
        go = bar * w + lam * wd;
        aa = lam * w;
      } else if (MODE == BOND) {
        const size_t bi = (size_t)s_idx[TM + row], bj = (size_t)s_idx[2 * TM + row];
        const float4 wi = ldg4(a.wgt + bi * 64 + c0), wj = ldg4(a.wgt + bj * 64 + c0);
        const float4 wdi = ldg4(a.wgt_d + bi * 64 + c0), wdj = ldg4(a.wgt_d + bj * 64 + c0);
        if (valid) {
          stg4(a.bar_w0 + (size_t)g * 64 + c0, bar * o * wj + lam * (od * wj + o * wdj));
          stg4(a.bar_w1 + (size_t)g * 64 + c0, bar * o * wi + lam * (od * wi + o * wdi));
        }
        go = bar * wi * wj + lam * (wdi * wj + wi * wdj);
        aa = lam * wi * wj;
      } else {
        go = bar;
        aa = lam;
      }
      float gy1[4], gy2[4], k1[4], k2[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float gj = f4at(go, j), aj = f4at(aa, j);
        const float dt = t[j] * (1.f - t[j]);
        const float d2s = d2silu_f(bc.y[j]);
        const float d2t = dt * (1.f - 2.f * t[j]);
        gy1[j] = gj * t[j] * dcore[j] + aj * (d2s * t[j] * bc.yd[j] + dcore[j] * dt * bg.yd[j]);
        gy2[j] = gj * core[j] * dt + aj * (dcore[j] * dt * bc.yd[j] + core[j] * d2t * bg.yd[j]);
        k1[j] = aj * dcore[j] * t[j];
        k2[j] = aj * core[j] * dt;
      }
      float q1[4], q2[4];
      branch_bwd2(bc, gy1, k1, use_ln, g1, q1, ln_acc, ln_acc + 4, valid);
      branch_bwd2(bg, gy2, k2, use_ln, g2, q2, ln_acc + 8, ln_acc + 12, valid);
      const float4 uc = make_float4(q1[0], q1[1], q1[2], q1[3]), ug = make_float4(q2[0], q2[1], q2[2], q2[3]);
      if (L::HAS_W2) {
        if (valid) {
          stg4(a.u_out + (size_t)g * 128 + c0, uc);
          stg4(a.u_out + (size_t)g * 128 + 64 + c0, ug);
        }
        sts4(s_g + row * HS + c0, uc);
        sts4(s_g + row * HS + 64 + c0, ug);
      } else if (valid) {  // no hidden layer: p == pre
        stg4(a.bar_pre + (size_t)g * 128 + c0, uc);
        stg4(a.bar_pre + (size_t)g * 128 + 64 + c0, ug);
      }
    }
    if (L::HAS_W2) {
      __syncthreads();
      float acc1[4][8], acc2[4][8];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc1[i][j] = acc2[i][j] = 0.f;
      gemm_blockdiag(acc1, s_g, s_w2, s_w2 + 64 * 64, 64, r0, c0);  // W2^T u
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const size_t r = (size_t)min(base + r0 + i, a.n_rows - 1);
        sts4(s_g + (r0 + i) * HS + c0, ldg4(a.g_p_lam + r * 128 + c0));
        sts4(s_g + (r0 + i) * HS + 64 + c0, ldg4(a.g_p_lam + r * 128 + 64 + c0));
      }
      __syncthreads();
      gemm_blockdiag(acc2, s_g, s_w2, s_w2 + 64 * 64, 64, r0, c0);  // W2^T g_p_lam
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int g = base + r0 + i;
        if (g >= a.n_rows) continue;
        float prc[4], prg[4], pdc[4], pdg[4];
        load8(a.save_pre, (size_t)g, c0, prc, prg);
        load8(a.pre_d, (size_t)g, c0, pdc, pdg);
        float4 oc, og;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          f4at(oc, j) = fmaf(dsilu_f(prc[j]), acc1[i][j], d2silu_f(prc[j]) * pdc[j] * acc2[i][j]);
          f4at(og, j) = fmaf(dsilu_f(prg[j]), acc1[i][4 + j], d2silu_f(prg[j]) * pdg[j] * acc2[i][4 + j]);
        }
        stg4(a.bar_pre + (size_t)g * 128 + c0, oc);
        stg4(a.bar_pre + (size_t)g * 128 + 64 + c0, og);
      }
    }
  }
  if (use_ln && a.g_ln != nullptr) {
    __syncthreads();
    float* s_red = smem;  // [16 ty][256]
#pragma unroll
    for (int which = 0; which < 4; ++which)
#pragma unroll
      for (int j = 0; j < 4; ++j) s_red[ty * 256 + which * 64 + c0 + j] = ln_acc[which * 4 + j];
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int r = 0; r < 16; ++r) tot += s_red[r * 256 + tid];
    atomicAdd(a.g_ln + tid, (double)tot);
  }
}

template <int MODE>
int launch_tan(const TanArgs& a, cudaStream_t stream) {
  if (a.n_rows == 0) return CHG_OK;
  constexpr int smem = TanSmem<MODE>::TOTAL_BYTES;
  static int slots_of[MAX_DEVICES] = {};  // per device: the attribute belongs to its context
  int& slots = slots_of[device_ordinal()];
  if (slots == 0) {
    CHG_CUDA(cudaFuncSetAttribute(gated_tan_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    slots = resident_ctas(gated_tan_kernel<MODE>, smem);
  }
  const int n_tiles = (a.n_rows + TM - 1) / TM;
  gated_tan_kernel<MODE><<<min(n_tiles, slots), NTHR, smem, stream>>>(a);
  CHG_LAUNCH_END();
}

template <int MODE>
int launch_bwd2(const Bwd2Args& a, cudaStream_t stream) {
  if (a.n_rows == 0) return CHG_OK;
  constexpr int smem = Bwd2Smem<MODE>::TOTAL_BYTES;
  static int slots_of[MAX_DEVICES] = {};  // per device: the attribute belongs to its context
  int& slots = slots_of[device_ordinal()];
  if (slots == 0) {
    CHG_CUDA(cudaFuncSetAttribute(gated_bwd2_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    slots = resident_ctas(gated_bwd2_kernel<MODE>, smem);
  }
  const int n_tiles = (a.n_rows + TM - 1) / TM;
  gated_bwd2_kernel<MODE><<<min(n_tiles, slots), NTHR, smem, stream>>>(a);
  CHG_LAUNCH_END();
}

}  // namespace
}  // namespace chg

using namespace chg;
using namespace chg::gated;

extern "C" int chg_atom_conv_tan(const float* pcn_d, const float* pe_d, const float* wag, const float* wag_d,
                                 const int32_t* center, const int32_t* nbr, const int32_t* d2u, int32_t n_edges,
                                 const float* save_pre, const float* save_p, const float* w2t, const float* ln,
                                 float* msg_d, float* pre_d, float* p_d, void* stream) {
  CHG_CHECK_ARG(n_edges >= 0, "negative size");
  if (n_edges == 0) return CHG_OK;
  CHG_CHECK_ARG(pcn_d && pe_d && wag && wag_d && center && nbr && d2u && save_pre && save_p && w2t && msg_d && pre_d && p_d,
                "null pointer");
  TanArgs a{pcn_d, pe_d, nullptr, nullptr, wag, wag_d, center, nbr, d2u, n_edges, save_pre, save_p, w2t, ln, msg_d, pre_d, p_d};
  return launch_tan<ATOM>(a, as_stream(stream));
}

extern "C" int chg_atom_conv_bwd2(const float* save_pre, const float* save_p, const float* pre_d, const float* p_d,
                                  const float* g_p_lam, const float* wag, const float* wag_d, const int32_t* center,
                                  const int32_t* d2u, int32_t n_edges, const float* lam_agg, const float* bar_agg,
                                  const float* w2, const float* ln, float* bar_pre, float* bar_w, float* u_out,
                                  double* g_ln, void* stream) {
  CHG_CHECK_ARG(n_edges >= 0, "negative size");
  if (n_edges == 0) return CHG_OK;
  CHG_CHECK_ARG(save_pre && save_p && pre_d && p_d && g_p_lam && wag && wag_d && center && d2u && lam_agg && bar_agg && w2 &&
                    bar_pre && bar_w && u_out, "null pointer");
  Bwd2Args a{save_pre, save_p, pre_d, p_d, g_p_lam, wag, wag_d, center, d2u, nullptr, n_edges, lam_agg, bar_agg, w2, ln,
             bar_pre, bar_w, nullptr, u_out, g_ln};
  return launch_bwd2<ATOM>(a, as_stream(stream));
}

extern "C" int chg_bond_conv_tan(const float* pij_d, const float* px_d, const float* pa_d, const float* wbg,
                                 const float* wbg_d, const int32_t* ang_atom, const int32_t* ang_i, const int32_t* ang_j,
                                 int32_t n_angles, const float* save_pre, const float* save_p, const float* w2t,
                                 const float* ln, float* upd_d, float* pre_d, float* p_d, void* stream) {
  CHG_CHECK_ARG(n_angles >= 0, "negative size");
  if (n_angles == 0) return CHG_OK;
  CHG_CHECK_ARG(pij_d && px_d && pa_d && wbg && wbg_d && ang_atom && ang_i && ang_j && save_pre && save_p && w2t && upd_d &&
                    pre_d && p_d, "null pointer");
  TanArgs a{pij_d, px_d, pa_d, nullptr, wbg, wbg_d, ang_i, ang_j, ang_atom, n_angles, save_pre, save_p, w2t, ln, upd_d, pre_d, p_d};
  return launch_tan<BOND>(a, as_stream(stream));
}

extern "C" int chg_bond_conv_bwd2(const float* save_pre, const float* save_p, const float* pre_d, const float* p_d,
                                  const float* g_p_lam, const float* wbg, const float* wbg_d, const int32_t* ang_i,
                                  const int32_t* ang_j, int32_t n_angles, const float* lam_agg, const float* bar_agg,
                                  const float* w2, const float* ln, float* bar_pre, float* bar_wi, float* bar_wj,
                                  float* u_out, double* g_ln, void* stream) {
  CHG_CHECK_ARG(n_angles >= 0, "negative size");
  if (n_angles == 0) return CHG_OK;
  CHG_CHECK_ARG(save_pre && save_p && pre_d && p_d && g_p_lam && wbg && wbg_d && ang_i && ang_j && lam_agg && bar_agg && w2 &&
                    bar_pre && bar_wi && bar_wj && u_out, "null pointer");
  Bwd2Args a{save_pre, save_p, pre_d, p_d, g_p_lam, wbg, wbg_d, ang_i, ang_i, ang_j, n_angles, lam_agg, bar_agg, w2, ln,
             bar_pre, bar_wi, bar_wj, u_out, g_ln};
  return launch_bwd2<BOND>(a, as_stream(stream));
}

extern "C" int chg_angle_update_tan(const float* pij_d, const float* px_d, const float* pa_d, const float* ang_d,
                                    const int32_t* ang_atom, const int32_t* ang_i, const int32_t* ang_j,
                                    int32_t n_angles, const float* save_p, const float* ln, float* ang_new_d, float* p_d,
                                    void* stream) {
  CHG_CHECK_ARG(n_angles >= 0, "negative size");
  if (n_angles == 0) return CHG_OK;
  CHG_CHECK_ARG(pij_d && px_d && pa_d && ang_d && ang_atom && ang_i && ang_j && save_p && ang_new_d && p_d, "null pointer");
  TanArgs a{pij_d, px_d, pa_d, ang_d, nullptr, nullptr, ang_i, ang_j, ang_atom, n_angles, nullptr, save_p, nullptr, ln,
            ang_new_d, nullptr, p_d};
  return launch_tan<ANGLE>(a, as_stream(stream));
}

extern "C" int chg_angle_update_bwd2(const float* save_p, const float* p_d, const float* lam_ang, const float* bar_ang,
                                     int32_t n_angles, const float* ln, float* bar_pre, double* g_ln, void* stream) {
  CHG_CHECK_ARG(n_angles >= 0, "negative size");
  if (n_angles == 0) return CHG_OK;
  CHG_CHECK_ARG(save_p && p_d && bar_pre, "null pointer");
  Bwd2Args a{nullptr, save_p, nullptr, p_d, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, n_angles, lam_ang, bar_ang,
             nullptr, ln, bar_pre, nullptr, nullptr, nullptr, g_ln};
  return launch_bwd2<ANGLE>(a, as_stream(stream));
}
