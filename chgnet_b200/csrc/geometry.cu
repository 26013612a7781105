// Geometry, basis expansion (+ fused 31->64 embeddings), their reverse, and the
// force / virial accumulation.  One warp per bond / angle; lanes own basis functions
// in the expansion phase and feature columns (lane, lane+32) in the embedding phase.
//
// Reference: chgnet/model/model.py:826-877 (BatchedGraph.from_graphs geometry),
// encoders.py:98-110, 144-146, basis.py:33-40, 108-116, 188-205, model.py:432-439,
// and the two autograd.grad calls of model.py:517-535 (here one analytic pass).
#include "common.cuh"

namespace chg {
namespace {

constexpr int MAX_BASIS = 32;  // radial <= 32, angular (2F+1) <= 32 : one lane per basis function

__global__ void embed_atoms_kernel(const int32_t* __restrict__ z, const float* __restrict__ emb, int n_atoms,
                                   float* __restrict__ x) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // one float4 per thread
  const int atom = idx >> 4, c4 = idx & 15;
  if (atom >= n_atoms) return;
  const int row = z[atom] - 1;
  // Z outside [1, 94]: the host raises IndexError before launching (batch.py, reference tests/test_encoders.py:25-28);
  // a raw C-ABI caller gets NaN features instead of an out-of-bounds read
  const float qnan = __int_as_float(0x7fc00000);
  const float4 v = (row >= 0 && row < CHG_MAX_Z) ? ldg4(emb + (size_t)row * 64 + c4 * 4) : make_float4(qnan, qnan, qnan, qnan);
  stg4(x + (size_t)atom * 64 + c4 * 4, v);
}

__global__ void edge_geometry_kernel(const float* __restrict__ frac, const float* __restrict__ lattice,
                                     const int32_t* __restrict__ owner, const int32_t* __restrict__ center,
                                     const int32_t* __restrict__ nbr, const float* __restrict__ image, int n_edges,
                                     float* __restrict__ rvec, float* __restrict__ dist, float* __restrict__ rhat) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const int c = center[e], n = nbr[e];
  const float* L = lattice + (size_t)owner[c] * 9;
  float l[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) l[i] = __ldg(L + i);
  const float fc[3] = {frac[c * 3], frac[c * 3 + 1], frac[c * 3 + 2]};
  const float fn[3] = {frac[n * 3], frac[n * 3 + 1], frac[n * 3 + 2]};
  const float im[3] = {image[(size_t)e * 3], image[(size_t)e * 3 + 1], image[(size_t)e * 3 + 2]};
  float r[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    // cart = frac @ L ; r = x_c - (x_n + img @ L)      (model.py:840, encoders.py:98-99)
    const float xc = fmaf(fc[2], l[6 + j], fmaf(fc[1], l[3 + j], fc[0] * l[j]));
    const float xn = fmaf(fn[2], l[6 + j], fmaf(fn[1], l[3 + j], fn[0] * l[j]));
    const float sh = fmaf(im[2], l[6 + j], fmaf(im[1], l[3 + j], im[0] * l[j]));
    r[j] = xc - (xn + sh);
  }
  const float d = sqrtf(fmaf(r[2], r[2], fmaf(r[1], r[1], r[0] * r[0])));
  dist[e] = d;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    rvec[(size_t)e * 3 + j] = r[j];
    rhat[(size_t)e * 3 + j] = r[j] / d;  // d == 0 -> NaN, as in the reference (tests/test_encoders.py:83-96)
  }
}

struct Envelope {
  float env, denv;  // value and d/dd
};
// polynomial cutoff 1 + a x^p + b x^(p+1) + c x^(p+2), x = d/rc < 1 (basis.py:184-205)
__device__ __forceinline__ Envelope envelope(float d, float rc, int p) {
  Envelope o;
  if (p == 0) {
    o.env = 1.f;
    o.denv = 0.f;
    return o;
  }
  const float x = d / rc;
  if (!(x < 1.f)) {
    o.env = 0.f;
    o.denv = 0.f;
    return o;
  }
  const float pf = (float)p;
  const float a = -(pf + 1.f) * (pf + 2.f) * 0.5f, b = pf * (pf + 2.f), c = -pf * (pf + 1.f) * 0.5f;
  float xp1 = 1.f;  // x^(p-1)
  for (int i = 0; i < p - 1; ++i) xp1 *= x;
  const float xp = xp1 * x;
  o.env = 1.f + xp * (a + x * (b + x * c));
  o.denv = xp1 * (a * pf + x * (b * (pf + 1.f) + x * c * (pf + 2.f))) / rc;
  return o;
}

// ---- bond basis + embeddings ---------------------------------------------------
__global__ void __launch_bounds__(256)
bond_basis_embed_kernel(const float* __restrict__ dist, const int32_t* __restrict__ u2d, int n_bonds,
                        const float* __restrict__ freq_ag, const float* __restrict__ freq_bg, int R, float rc_ag,
                        float rc_bg, int p, const float* __restrict__ w3t, float* __restrict__ e0,
                        float* __restrict__ wag, float* __restrict__ wbg, float* __restrict__ basis_out) {
  extern __shared__ __align__(16) float s_w[];  // [3][R][64]
  for (int i = threadIdx.x; i < 3 * R * 64; i += blockDim.x) s_w[i] = w3t[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  const float f_ag = lane < R ? freq_ag[lane] : 0.f;
  const float f_bg = lane < R ? freq_bg[lane] : 0.f;
  const float nrm_ag = sqrtf(2.f / rc_ag), nrm_bg = sqrtf(2.f / rc_bg);
  const float inv_ag = 1.f / rc_ag, inv_bg = 1.f / rc_bg;  // basis.py:108 multiplies by 1/cutoff
  // IT bonds per warp iteration: the weight rows read from shared memory are reused IT times and
  // the IT x 6 accumulators give the FMA pipe independent work
  constexpr int IT = 4;
  for (int u0 = warp * IT; u0 < n_bonds; u0 += n_warps * IT) {
    float b_ag[IT], b_bg[IT];
    bool bg_live = false;  // warp-uniform
#pragma unroll
    for (int q = 0; q < IT; ++q) {
      const float d = dist[u2d[min(u0 + q, n_bonds - 1)]];
      const Envelope ea = envelope(d, rc_ag, p), eb = envelope(d, rc_bg, p);
      // basis.py:110: norm * sin(freq * d_scaled) / d * envelope
      b_ag[q] = lane < R ? ea.env * (nrm_ag * sinf(f_ag * (d * inv_ag)) / d) : 0.f;
      b_bg[q] = lane < R ? eb.env * (nrm_bg * sinf(f_bg * (d * inv_bg)) / d) : 0.f;
      bg_live = bg_live || eb.env != 0.f || !(d == d);  // NaN propagates
      if (basis_out != nullptr && u0 + q < n_bonds) {  // training: [ag basis | bg basis], 32 columns each
        basis_out[(size_t)(u0 + q) * 64 + lane] = b_ag[q];
        basis_out[(size_t)(u0 + q) * 64 + 32 + lane] = b_bg[q];
      }
    }
    float o[IT][6];
#pragma unroll
    for (int q = 0; q < IT; ++q)
#pragma unroll
      for (int j = 0; j < 6; ++j) o[q][j] = 0.f;
    for (int k = 0; k < R; ++k) {
      const float* w = s_w + k * 64;
      const float w0a = w[lane], w0b = w[lane + 32], w1a = w[R * 64 + lane], w1b = w[R * 64 + lane + 32];
#pragma unroll
      for (int q = 0; q < IT; ++q) {
        const float ba = __shfl_sync(0xffffffffu, b_ag[q], k);
        o[q][0] = fmaf(ba, w0a, o[q][0]);
        o[q][1] = fmaf(ba, w0b, o[q][1]);
        o[q][2] = fmaf(ba, w1a, o[q][2]);
        o[q][3] = fmaf(ba, w1b, o[q][3]);
      }
      if (bg_live) {
        const float w2a = w[2 * R * 64 + lane], w2b = w[2 * R * 64 + lane + 32];
#pragma unroll
        for (int q = 0; q < IT; ++q) {
          const float bb = __shfl_sync(0xffffffffu, b_bg[q], k);
          o[q][4] = fmaf(bb, w2a, o[q][4]);
          o[q][5] = fmaf(bb, w2b, o[q][5]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < IT; ++q) {
      const int u = u0 + q;
      if (u < n_bonds) {
        float* r0 = e0 + (size_t)u * 64;
        float* r1 = wag + (size_t)u * 64;
        float* r2 = wbg + (size_t)u * 64;
        r0[lane] = o[q][0]; r0[lane + 32] = o[q][1];
        r1[lane] = o[q][2]; r1[lane + 32] = o[q][3];
        r2[lane] = o[q][4]; r2[lane + 32] = o[q][5];
      }
    }
  }
}

__global__ void __launch_bounds__(256)
bond_basis_bwd_kernel(const float* __restrict__ dist, const int32_t* __restrict__ u2d, int n_bonds,
                      const float* __restrict__ freq_ag, const float* __restrict__ freq_bg, int R, float rc_ag,
                      float rc_bg, int p, const float* __restrict__ w3, const float* __restrict__ g_e0,
                      const float* __restrict__ g_wag, const float* __restrict__ g_wbg,
                      float* __restrict__ g_dist, double* __restrict__ g_freq) {
  extern __shared__ __align__(16) float s_w[];  // [3][64][R]
  for (int i = threadIdx.x; i < 3 * R * 64; i += blockDim.x) s_w[i] = w3[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  const int kl = lane < R ? lane : 0;
  const float f_ag = freq_ag[kl], f_bg = freq_bg[kl];
  const float nrm_ag = sqrtf(2.f / rc_ag), nrm_bg = sqrtf(2.f / rc_bg);
  constexpr int IT = 2;  // bonds per warp iteration
  double gf_ag = 0.0, gf_bg = 0.0;  // training: lane k accumulates dL/d freq_k
  for (int u0 = warp * IT; u0 < n_bonds; u0 += n_warps * IT) {
    float d[IT], a0[IT], a1[IT], b0[IT], b1[IT], c0[IT], c1[IT];
    Envelope ea[IT], eb[IT];
    bool bg_live = false;
#pragma unroll
    for (int q = 0; q < IT; ++q) {
      const int u = min(u0 + q, n_bonds - 1);
      d[q] = dist[u2d[u]];
      ea[q] = envelope(d[q], rc_ag, p);
      eb[q] = envelope(d[q], rc_bg, p);
      const float* q0 = g_e0 + (size_t)u * 64;
      const float* q1 = g_wag + (size_t)u * 64;
      const float* q2 = g_wbg + (size_t)u * 64;
      a0[q] = q0[lane]; a1[q] = q0[lane + 32];
      b0[q] = q1[lane]; b1[q] = q1[lane + 32];
      c0[q] = q2[lane]; c1[q] = q2[lane + 32];
      bg_live = bg_live || eb[q].env != 0.f || eb[q].denv != 0.f || !(d[q] == d[q]);
    }
    // lane k: gradient wrt basis function k
    float gb_ag[IT], gb_bg[IT];
#pragma unroll
    for (int q = 0; q < IT; ++q) gb_ag[q] = gb_bg[q] = 0.f;
    for (int n = 0; n < 32; ++n) {
      const float w00 = s_w[n * R + kl], w01 = s_w[(n + 32) * R + kl];
      const float w10 = s_w[(64 + n) * R + kl], w11 = s_w[(64 + n + 32) * R + kl];
#pragma unroll
      for (int q = 0; q < IT; ++q) {
        gb_ag[q] = fmaf(__shfl_sync(0xffffffffu, a0[q], n), w00, gb_ag[q]);
        gb_ag[q] = fmaf(__shfl_sync(0xffffffffu, b0[q], n), w10, gb_ag[q]);
        gb_ag[q] = fmaf(__shfl_sync(0xffffffffu, a1[q], n), w01, gb_ag[q]);
        gb_ag[q] = fmaf(__shfl_sync(0xffffffffu, b1[q], n), w11, gb_ag[q]);
      }
      if (bg_live) {
        const float w20 = s_w[(128 + n) * R + kl], w21 = s_w[(128 + n + 32) * R + kl];
#pragma unroll
        for (int q = 0; q < IT; ++q) {
          gb_bg[q] = fmaf(__shfl_sync(0xffffffffu, c0[q], n), w20, gb_bg[q]);
          gb_bg[q] = fmaf(__shfl_sync(0xffffffffu, c1[q], n), w21, gb_bg[q]);
        }
      }
    }
    // d basis_k / dd = norm [ (w/rc) cos(w d/rc)/d - sin(w d/rc)/d^2 ] env + norm sin(w d/rc)/d env'
#pragma unroll
    for (int q = 0; q < IT; ++q) {
      float contrib = 0.f;
      if (lane < R) {
        float sn, cs;
        sincosf(f_ag * (d[q] / rc_ag), &sn, &cs);
        const float raw = nrm_ag * sn / d[q];
        const float draw = nrm_ag * ((f_ag / rc_ag) * cs / d[q] - sn / (d[q] * d[q]));
        contrib = gb_ag[q] * fmaf(draw, ea[q].env, raw * ea[q].denv);
        const bool live_q = u0 + q < n_bonds;
        // d basis_k / d freq_k = norm cos(w d/rc) / rc * env
        if (g_freq != nullptr && live_q) gf_ag += (double)(gb_ag[q] * (nrm_ag * cs / rc_ag) * ea[q].env);
        if (eb[q].env != 0.f || eb[q].denv != 0.f || !(d[q] == d[q])) {
          sincosf(f_bg * (d[q] / rc_bg), &sn, &cs);
          if (g_freq != nullptr && live_q) gf_bg += (double)(gb_bg[q] * (nrm_bg * cs / rc_bg) * eb[q].env);
          const float raw2 = nrm_bg * sn / d[q];
          const float draw2 = nrm_bg * ((f_bg / rc_bg) * cs / d[q] - sn / (d[q] * d[q]));
          contrib += gb_bg[q] * fmaf(draw2, eb[q].env, raw2 * eb[q].denv);
        }
      }
      contrib = sum32(contrib);
      if (lane == 0 && u0 + q < n_bonds) g_dist[u0 + q] = contrib;
    }
  }
  if (g_freq != nullptr && lane < R) {
    atomicAdd(g_freq + lane, gf_ag);
    atomicAdd(g_freq + R + lane, gf_bg);
  }
}

// ---- angle basis + embedding -----------------------------------------------------
__device__ __forceinline__ float angle_cos(const float* __restrict__ rhat, int di, int dj, float (&ri)[3],
                                           float (&rj)[3]) {
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    ri[j] = rhat[(size_t)di * 3 + j];
    rj[j] = rhat[(size_t)dj * 3 + j];
  }
  // encoders.py:144: (1 - 1e-6) keeps acos away from |u| = 1
  return fmaf(ri[2], rj[2], fmaf(ri[1], rj[1], ri[0] * rj[0])) * (1.f - 1e-6f);
}

__global__ void __launch_bounds__(256)
angle_basis_embed_kernel(const float* __restrict__ rhat, const int32_t* __restrict__ ang_di,
                         const int32_t* __restrict__ ang_dj, int n_angles, const float* __restrict__ freq, int nf,
                         const float* __restrict__ wt, float* __restrict__ a0, float* __restrict__ basis_out) {
  extern __shared__ __align__(16) float s_w[];  // [2nf+1][64]
  const int nb = 2 * nf + 1;
  for (int i = threadIdx.x; i < nb * 64; i += blockDim.x) s_w[i] = wt[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  const bool is_sin = lane >= 1 && lane <= nf, is_cos = lane > nf && lane < nb;
  const float w = is_sin ? freq[lane - 1] : (is_cos ? freq[lane - 1 - nf] : 0.f);
  const float inv_sqrt_pi = 0.5641895835477563f;
  constexpr int IT = 4;  // angles per warp iteration (weight rows reused, independent accumulators)
  for (int a0i = warp * IT; a0i < n_angles; a0i += n_warps * IT) {
    float f[IT];
#pragma unroll
    for (int q = 0; q < IT; ++q) {
      const int a = min(a0i + q, n_angles - 1);
      float ri[3], rj[3];
      const float u = angle_cos(rhat, ang_di[a], ang_dj[a], ri, rj);
      const float th = acosf(u);
      float v = 0.f;
      if (lane == 0) v = 0.7071067811865476f;
      else if (is_sin) v = sinf(w * th);
      else if (is_cos) v = cosf(w * th);
      f[q] = v * inv_sqrt_pi;
      if (basis_out != nullptr && a0i + q < n_angles) {  // training: basis in columns 0..2nf, zeros after
        basis_out[(size_t)(a0i + q) * 64 + lane] = f[q];
        basis_out[(size_t)(a0i + q) * 64 + 32 + lane] = 0.f;
      }
    }
    float oa[IT], ob[IT];
#pragma unroll
    for (int q = 0; q < IT; ++q) oa[q] = ob[q] = 0.f;
    for (int m = 0; m < nb; ++m) {
      const float wa = s_w[m * 64 + lane], wb = s_w[m * 64 + lane + 32];
#pragma unroll
      for (int q = 0; q < IT; ++q) {
        const float fm = __shfl_sync(0xffffffffu, f[q], m);
        oa[q] = fmaf(fm, wa, oa[q]);
        ob[q] = fmaf(fm, wb, ob[q]);
      }
    }
#pragma unroll
    for (int q = 0; q < IT; ++q) {
      const int a = a0i + q;
      if (a < n_angles) {
        a0[(size_t)a * 64 + lane] = oa[q];
        a0[(size_t)a * 64 + lane + 32] = ob[q];
      }
    }
  }
}

__global__ void __launch_bounds__(256)
angle_basis_bwd_kernel(const float* __restrict__ rhat, const int32_t* __restrict__ ang_di,
                       const int32_t* __restrict__ ang_dj, int n_angles, const float* __restrict__ freq, int nf,
                       const float* __restrict__ w, const float* __restrict__ g_a0, double* __restrict__ g_rhat,
                       double* __restrict__ g_freq) {
  extern __shared__ __align__(16) float s_w[];  // [64][2nf+1]
  const int nb = 2 * nf + 1;
  for (int i = threadIdx.x; i < nb * 64; i += blockDim.x) s_w[i] = w[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  const bool is_sin = lane >= 1 && lane <= nf, is_cos = lane > nf && lane < nb;
  const float wf = is_sin ? freq[lane - 1] : (is_cos ? freq[lane - 1 - nf] : 0.f);
  const int ml = lane < nb ? lane : 0;
  const float inv_sqrt_pi = 0.5641895835477563f;
  // A warp owns CHUNK consecutive angles.  Angles are sorted by bond i, so the directed edge
  // di repeats in runs: its contribution is accumulated in registers and flushed with one
  // atomic per component when di changes (cuts same-address fp64 atomics by the run length).
  constexpr int CHUNK = 16;
  const int n_chunks = (n_angles + CHUNK - 1) / CHUNK;
  double gfr = 0.0;  // training: sin lane k and cos lane k both accumulate into dL/d freq_k
  for (int ch = warp; ch < n_chunks; ch += n_warps) {
    const int a_beg = ch * CHUNK, a_end = min(a_beg + CHUNK, n_angles);
    int cur_di = -1;
    double acc_i = 0.0;  // lanes 0..2: pending sum for g_rhat[cur_di][lane]
    for (int a = a_beg; a < a_end; a += 2) {  // two angles per pass share the weight reads
      const int a2 = min(a + 1, a_end - 1);
      const int di[2] = {ang_di[a], ang_di[a2]}, dj[2] = {ang_dj[a], ang_dj[a2]};
      float ri[2][3], rj[2][3], u[2], th[2], ga[2], gb[2], gf[2] = {0.f, 0.f};
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int aa = q == 0 ? a : a2;
        u[q] = angle_cos(rhat, di[q], dj[q], ri[q], rj[q]);
        th[q] = acosf(u[q]);
        ga[q] = g_a0[(size_t)aa * 64 + lane];
        gb[q] = g_a0[(size_t)aa * 64 + lane + 32];
      }
      for (int n = 0; n < 32; ++n) {  // lane m: dE/d f_m
        const float w0 = s_w[n * nb + ml], w1 = s_w[(n + 32) * nb + ml];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          gf[q] = fmaf(__shfl_sync(0xffffffffu, ga[q], n), w0, gf[q]);
          gf[q] = fmaf(__shfl_sync(0xffffffffu, gb[q], n), w1, gf[q]);
        }
      }
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        if (q == 1 && a + 1 >= a_end) break;  // warp-uniform
        float g_th = 0.f;
        if (is_sin) g_th = gf[q] * wf * cosf(wf * th[q]);
        else if (is_cos) g_th = -gf[q] * wf * sinf(wf * th[q]);
        if (g_freq != nullptr) {  // d sin(w th)/dw = th cos(w th), d cos(w th)/dw = -th sin(w th)
          if (is_sin) gfr += (double)(gf[q] * th[q] * cosf(wf * th[q]) * inv_sqrt_pi);
          else if (is_cos) gfr -= (double)(gf[q] * th[q] * sinf(wf * th[q]) * inv_sqrt_pi);
        }
        g_th = sum32(g_th) * inv_sqrt_pi;
        if (g_rhat == nullptr) continue;
        // d theta / d u' = -1/sqrt(1-u'^2); u' = (1-1e-6) u
        const float g_u = -g_th / sqrtf(1.f - u[q] * u[q]) * (1.f - 1e-6f);
        if (di[q] != cur_di) {
          if (cur_di >= 0 && lane < 3) atomicAdd(g_rhat + (size_t)cur_di * 3 + lane, acc_i);
          cur_di = di[q];
          acc_i = 0.0;
        }
        if (lane < 3) acc_i += (double)(g_u * rj[q][lane]);
        else if (lane < 6) atomicAdd(g_rhat + (size_t)dj[q] * 3 + (lane - 3), (double)(g_u * ri[q][lane - 3]));
      }
    }
    if (g_rhat != nullptr && cur_di >= 0 && lane < 3) atomicAdd(g_rhat + (size_t)cur_di * 3 + lane, acc_i);
  }
  if (g_freq != nullptr) {
    if (is_sin) atomicAdd(g_freq + lane - 1, gfr);
    else if (is_cos) atomicAdd(g_freq + lane - 1 - nf, gfr);
  }
}

// =====================================================================================
// Second-order pass of a force / stress loss (reference model.py:518-535 create_graph=True):
// tangents along a fixed direction rdot of the edge vectors, and the mixed derivatives of the
// basis functions with respect to their learnable frequencies.
// =====================================================================================
__global__ void edge_tangent_kernel(const float* __restrict__ rvec, const float* __restrict__ dist,
                                    const float* __restrict__ rhat, const int32_t* __restrict__ center,
                                    const int32_t* __restrict__ nbr, const int32_t* __restrict__ owner,
                                    const float* __restrict__ u_atom, const float* __restrict__ w_graph, int n_edges,
                                    float* __restrict__ ddist, float* __restrict__ drhat) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const int c = center[e], n = nbr[e];
  const float* W = w_graph + (size_t)owner[c] * 9;
  float r[3], rh[3], rd[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    r[j] = rvec[(size_t)e * 3 + j];
    rh[j] = rhat[(size_t)e * 3 + j];
  }
#pragma unroll
  for (int j = 0; j < 3; ++j)  // rdot = u[c] - u[n] + r . W
    rd[j] = u_atom[(size_t)c * 3 + j] - u_atom[(size_t)n * 3 + j] +
            fmaf(r[2], __ldg(W + 6 + j), fmaf(r[1], __ldg(W + 3 + j), r[0] * __ldg(W + j)));
  const float dd = fmaf(rh[2], rd[2], fmaf(rh[1], rd[1], rh[0] * rd[0]));
  const float inv_d = 1.f / dist[e];
  ddist[e] = dd;
#pragma unroll
  for (int j = 0; j < 3; ++j) drhat[(size_t)e * 3 + j] = (rd[j] - rh[j] * dd) * inv_d;
}

// d basis_k / dd for lane k (0 outside the basis), both cutoffs
__device__ __forceinline__ void rbf_ddist(float d, float f_ag, float f_bg, float rc_ag, float rc_bg, int p, bool live,
                                          float& dag, float& dbg) {
  dag = dbg = 0.f;
  if (!live) return;
  const Envelope ea = envelope(d, rc_ag, p), eb = envelope(d, rc_bg, p);
  const float nrm_ag = sqrtf(2.f / rc_ag), nrm_bg = sqrtf(2.f / rc_bg);
  float sn, cs;
  sincosf(f_ag * (d / rc_ag), &sn, &cs);
  dag = fmaf(nrm_ag * ((f_ag / rc_ag) * cs / d - sn / (d * d)), ea.env, (nrm_ag * sn / d) * ea.denv);
  if (eb.env != 0.f || eb.denv != 0.f || !(d == d)) {
    sincosf(f_bg * (d / rc_bg), &sn, &cs);
    dbg = fmaf(nrm_bg * ((f_bg / rc_bg) * cs / d - sn / (d * d)), eb.env, (nrm_bg * sn / d) * eb.denv);
  }
}

__global__ void __launch_bounds__(256)
bond_basis_tangent_kernel(const float* __restrict__ dist, const float* __restrict__ ddist,
                          const int32_t* __restrict__ u2d, int n_bonds, const float* __restrict__ freq_ag,
                          const float* __restrict__ freq_bg, int R, float rc_ag, float rc_bg, int p,
                          const float* __restrict__ w3t, float* __restrict__ e0d, float* __restrict__ wagd,
                          float* __restrict__ wbgd, float* __restrict__ tbasis) {
  extern __shared__ __align__(16) float s_w[];  // [3][R][64]
  for (int i = threadIdx.x; i < 3 * R * 64; i += blockDim.x) s_w[i] = w3t[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  const float f_ag = lane < R ? freq_ag[lane] : 0.f, f_bg = lane < R ? freq_bg[lane] : 0.f;
  for (int u = warp; u < n_bonds; u += n_warps) {
    const int e = u2d[u];
    const float d = dist[e], dd = ddist[e];
    float tag, tbg;
    rbf_ddist(d, f_ag, f_bg, rc_ag, rc_bg, p, lane < R, tag, tbg);
    tag *= dd;
    tbg *= dd;
    tbasis[(size_t)u * 64 + lane] = tag;
    tbasis[(size_t)u * 64 + 32 + lane] = tbg;
    float o[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < R; ++k) {
      const float* w = s_w + k * 64;
      const float ba = __shfl_sync(0xffffffffu, tag, k), bb = __shfl_sync(0xffffffffu, tbg, k);
      o[0] = fmaf(ba, w[lane], o[0]);
      o[1] = fmaf(ba, w[lane + 32], o[1]);
      o[2] = fmaf(ba, w[R * 64 + lane], o[2]);
      o[3] = fmaf(ba, w[R * 64 + lane + 32], o[3]);
      o[4] = fmaf(bb, w[2 * R * 64 + lane], o[4]);
      o[5] = fmaf(bb, w[2 * R * 64 + lane + 32], o[5]);
    }
    e0d[(size_t)u * 64 + lane] = o[0];
    e0d[(size_t)u * 64 + lane + 32] = o[1];
    wagd[(size_t)u * 64 + lane] = o[2];
    wagd[(size_t)u * 64 + lane + 32] = o[3];
    wbgd[(size_t)u * 64 + lane] = o[4];
    wbgd[(size_t)u * 64 + lane + 32] = o[5];
  }
}

// d^2 envelope / dd^2 (basis.py:184-205 differentiated twice)
__device__ __forceinline__ float envelope_d2(float d, float rc, int p) {
  const float x = d / rc;
  if (p == 0 || !(x < 1.f)) return 0.f;
  const float pf = (float)p;
  const float a = -(pf + 1.f) * (pf + 2.f) * 0.5f, b = pf * (pf + 2.f), c = -pf * (pf + 1.f) * 0.5f;
  float xpm1 = 1.f;  // x^(p-1)
  for (int i = 0; i < p - 1; ++i) xpm1 *= x;
  float t0 = 0.f;  // a p (p-1) x^(p-2)
  if (p >= 2) {
    float xpm2 = 1.f;
    for (int i = 0; i < p - 2; ++i) xpm2 *= x;
    t0 = a * pf * (pf - 1.f) * xpm2;
  }
  return (t0 + xpm1 * (b * (pf + 1.f) * pf + x * c * (pf + 2.f) * (pf + 1.f))) / (rc * rc);
}

// d^2 basis / dd^2 of the basis function of frequency f:  raw'' env + 2 raw' env' + raw env''
__device__ __forceinline__ float rbf_d2(float d, float f, float rc, int p) {
  const Envelope e = envelope(d, rc, p);
  const float nrm = sqrtf(2.f / rc), k = f / rc;
  float sn, cs;
  sincosf(f * (d / rc), &sn, &cs);
  const float raw = nrm * sn / d;
  const float draw = nrm * (k * cs / d - sn / (d * d));
  const float d2raw = nrm * (-k * k * sn / d - 2.f * k * cs / (d * d) + 2.f * sn / (d * d * d));
  return d2raw * e.env + 2.f * draw * e.denv + raw * envelope_d2(d, rc, p);
}

// kGeom = false: g_freq += d/dfreq < lam, (dB/dd ddist) W >          (force / stress loss)
// kGeom = true : g_dist[u] += < lam W^T, d^2B/dd^2 > ddist             (Hessian-vector product)
template <bool kGeom>
__global__ void __launch_bounds__(256)
bond_basis_bwd2_kernel(const float* __restrict__ dist, const float* __restrict__ ddist,
                       const int32_t* __restrict__ u2d, int n_bonds, const float* __restrict__ freq_ag,
                       const float* __restrict__ freq_bg, int R, float rc_ag, float rc_bg, int p,
                       const float* __restrict__ w3, const float* __restrict__ lam_e0,
                       const float* __restrict__ lam_wag, const float* __restrict__ lam_wbg,
                       double* __restrict__ g_freq, float* __restrict__ g_dist) {
  extern __shared__ __align__(16) float s_w[];  // [3][64][R]
  for (int i = threadIdx.x; i < 3 * R * 64; i += blockDim.x) s_w[i] = w3[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  const int kl = lane < R ? lane : 0;
  const float f_ag = freq_ag[kl], f_bg = freq_bg[kl];
  const float nrm_ag = sqrtf(2.f / rc_ag), nrm_bg = sqrtf(2.f / rc_bg);
  double gf_ag = 0.0, gf_bg = 0.0;
  for (int u = warp; u < n_bonds; u += n_warps) {
    const int e = u2d[u];
    const float d = dist[e], dd = ddist[e];
    const float a0 = lam_e0[(size_t)u * 64 + lane], a1 = lam_e0[(size_t)u * 64 + lane + 32];
    const float b0 = lam_wag[(size_t)u * 64 + lane], b1 = lam_wag[(size_t)u * 64 + lane + 32];
    const float c0 = lam_wbg[(size_t)u * 64 + lane], c1 = lam_wbg[(size_t)u * 64 + lane + 32];
    float gb_ag = 0.f, gb_bg = 0.f;
    for (int n = 0; n < 32; ++n) {
      gb_ag = fmaf(__shfl_sync(0xffffffffu, a0, n), s_w[n * R + kl], gb_ag);
      gb_ag = fmaf(__shfl_sync(0xffffffffu, a1, n), s_w[(n + 32) * R + kl], gb_ag);
      gb_ag = fmaf(__shfl_sync(0xffffffffu, b0, n), s_w[(64 + n) * R + kl], gb_ag);
      gb_ag = fmaf(__shfl_sync(0xffffffffu, b1, n), s_w[(64 + n + 32) * R + kl], gb_ag);
      gb_bg = fmaf(__shfl_sync(0xffffffffu, c0, n), s_w[(128 + n) * R + kl], gb_bg);
      gb_bg = fmaf(__shfl_sync(0xffffffffu, c1, n), s_w[(128 + n + 32) * R + kl], gb_bg);
    }
    if constexpr (kGeom) {
      float src = 0.f;
      if (lane < R) {
        src = gb_ag * rbf_d2(d, f_ag, rc_ag, p);
        const Envelope eb = envelope(d, rc_bg, p);
        if (eb.env != 0.f || eb.denv != 0.f || !(d == d)) src = fmaf(gb_bg, rbf_d2(d, f_bg, rc_bg, p), src);
      }
      src = sum32(src);
      if (lane == 0) g_dist[u] += src * dd;  // one warp per bond: no other writer
    } else if (lane < R) {
      // d/dw of  nrm [ (w/rc) cos(w x)/d - sin(w x)/d^2 ] env + nrm sin(w x)/d env' ,  x = d/rc
      const Envelope ea = envelope(d, rc_ag, p), eb = envelope(d, rc_bg, p);
      float sn, cs;
      float x = d / rc_ag;
      sincosf(f_ag * x, &sn, &cs);
      float mixed = nrm_ag * (cs / (rc_ag * d) - (f_ag / rc_ag) * x * sn / d - x * cs / (d * d)) * ea.env +
                    nrm_ag * x * cs / d * ea.denv;
      gf_ag += (double)(gb_ag * mixed * dd);
      if (eb.env != 0.f || eb.denv != 0.f || !(d == d)) {
        x = d / rc_bg;
        sincosf(f_bg * x, &sn, &cs);
        mixed = nrm_bg * (cs / (rc_bg * d) - (f_bg / rc_bg) * x * sn / d - x * cs / (d * d)) * eb.env +
                nrm_bg * x * cs / d * eb.denv;
        gf_bg += (double)(gb_bg * mixed * dd);
      }
    }
  }
  if (!kGeom && lane < R) {
    atomicAdd(g_freq + lane, gf_ag);
    atomicAdd(g_freq + R + lane, gf_bg);
  }
}

// theta and its tangent for angle (di, dj)
__device__ __forceinline__ void theta_dot(const float* __restrict__ rhat, const float* __restrict__ drhat, int di,
                                          int dj, float& th, float& thd) {
  float ri[3], rj[3];
  const float u = angle_cos(rhat, di, dj, ri, rj);
  float ud = 0.f;
#pragma unroll
  for (int j = 0; j < 3; ++j)
    ud = fmaf(drhat[(size_t)di * 3 + j], rj[j], fmaf(ri[j], drhat[(size_t)dj * 3 + j], ud));
  ud *= (1.f - 1e-6f);
  th = acosf(u);
  thd = -ud / sqrtf(1.f - u * u);
}

__global__ void __launch_bounds__(256)
angle_basis_tangent_kernel(const float* __restrict__ rhat, const float* __restrict__ drhat,
                           const int32_t* __restrict__ ang_di, const int32_t* __restrict__ ang_dj, int n_angles,
                           const float* __restrict__ freq, int nf, const float* __restrict__ wt,
                           float* __restrict__ a0d, float* __restrict__ tbasis) {
  extern __shared__ __align__(16) float s_w[];  // [2nf+1][64]
  const int nb = 2 * nf + 1;
  for (int i = threadIdx.x; i < nb * 64; i += blockDim.x) s_w[i] = wt[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  const bool is_sin = lane >= 1 && lane <= nf, is_cos = lane > nf && lane < nb;
  const float w = is_sin ? freq[lane - 1] : (is_cos ? freq[lane - 1 - nf] : 0.f);
  const float inv_sqrt_pi = 0.5641895835477563f;
  for (int a = warp; a < n_angles; a += n_warps) {
    float th, thd;
    theta_dot(rhat, drhat, ang_di[a], ang_dj[a], th, thd);
    float fd = 0.f;
    if (is_sin) fd = w * cosf(w * th);
    else if (is_cos) fd = -w * sinf(w * th);
    fd *= thd * inv_sqrt_pi;
    tbasis[(size_t)a * 64 + lane] = fd;
    tbasis[(size_t)a * 64 + 32 + lane] = 0.f;
    float oa = 0.f, ob = 0.f;
    for (int m = 0; m < nb; ++m) {
      const float fm = __shfl_sync(0xffffffffu, fd, m);
      oa = fmaf(fm, s_w[m * 64 + lane], oa);
      ob = fmaf(fm, s_w[m * 64 + lane + 32], ob);
    }
    a0d[(size_t)a * 64 + lane] = oa;
    a0d[(size_t)a * 64 + lane + 32] = ob;
  }
}

// theta, its tangent, and what the geometry derivative of the tangent needs, with 1 - u^2 formed as
// (1 - c^2) + c^2 |rhat_i x rhat_j|^2: at an exactly collinear pair 1 - u^2 ~ 2e-6, and 1 - u*u in fp32
// would lose ~3 % of it to cancellation (d^2 theta carries its -3/2 power)
struct ThetaGeom {
  float ri[3], rj[3], dri[3], drj[3];
  float u, ud, th, th_u;  // u = c rhat_i . rhat_j, ud its tangent, th_u = d theta / du
};
__device__ __forceinline__ ThetaGeom theta_geom(const float* __restrict__ rhat, const float* __restrict__ drhat,
                                                int di, int dj) {
  ThetaGeom g;
  g.u = angle_cos(rhat, di, dj, g.ri, g.rj);
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    g.dri[j] = drhat[(size_t)di * 3 + j];
    g.drj[j] = drhat[(size_t)dj * 3 + j];
  }
  constexpr float c = 1.f - 1e-6f;
  const float x0 = g.ri[1] * g.rj[2] - g.ri[2] * g.rj[1], x1 = g.ri[2] * g.rj[0] - g.ri[0] * g.rj[2],
              x2 = g.ri[0] * g.rj[1] - g.ri[1] * g.rj[0];
  const float one_m_c2 = 1e-6f * (2.f - 1e-6f);
  const float q = fmaf(c * c, fmaf(x2, x2, fmaf(x1, x1, x0 * x0)), one_m_c2);
  float ud = 0.f;
#pragma unroll
  for (int j = 0; j < 3; ++j) ud = fmaf(g.dri[j], g.rj[j], fmaf(g.ri[j], g.drj[j], ud));
  g.ud = ud * c;
  g.th = acosf(g.u);
  g.th_u = -rsqrtf(q);
  return g;
}

__device__ __forceinline__ float pick3(const float (&v)[3], int k) { return k == 0 ? v[0] : (k == 1 ? v[1] : v[2]); }

// kGeom = false: g_freq += d/dfreq < lam_a0, (dF/dtheta thetadot) W >                     (force / stress loss)
// kGeom = true : g_rhat += d/d(rhat_i, rhat_j) < lam_a0, (dF/dtheta thetadot) W >, drhat fixed (Hessian-vector)
template <bool kGeom>
__global__ void __launch_bounds__(256)
angle_basis_bwd2_kernel(const float* __restrict__ rhat, const float* __restrict__ drhat,
                        const int32_t* __restrict__ ang_di, const int32_t* __restrict__ ang_dj, int n_angles,
                        const float* __restrict__ freq, int nf, const float* __restrict__ w,
                        const float* __restrict__ lam_a0, double* __restrict__ g_freq, double* __restrict__ g_rhat) {
  extern __shared__ __align__(16) float s_w[];  // [64][2nf+1]
  const int nb = 2 * nf + 1;
  for (int i = threadIdx.x; i < nb * 64; i += blockDim.x) s_w[i] = w[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  const bool is_sin = lane >= 1 && lane <= nf, is_cos = lane > nf && lane < nb;
  const float wf = is_sin ? freq[lane - 1] : (is_cos ? freq[lane - 1 - nf] : 0.f);
  const int ml = lane < nb ? lane : 0;
  const float inv_sqrt_pi = 0.5641895835477563f;
  double gfr = 0.0;
  for (int a = warp; a < n_angles; a += n_warps) {
    float th, thd;
    ThetaGeom tg;
    if constexpr (kGeom) {
      tg = theta_geom(rhat, drhat, ang_di[a], ang_dj[a]);
      th = tg.th;
      thd = tg.th_u * tg.ud;
    } else {
      theta_dot(rhat, drhat, ang_di[a], ang_dj[a], th, thd);
    }
    const float ga = lam_a0[(size_t)a * 64 + lane], gb = lam_a0[(size_t)a * 64 + lane + 32];
    float gf = 0.f;
    for (int n = 0; n < 32; ++n) {
      gf = fmaf(__shfl_sync(0xffffffffu, ga, n), s_w[n * nb + ml], gf);
      gf = fmaf(__shfl_sync(0xffffffffu, gb, n), s_w[(n + 32) * nb + ml], gf);
    }
    float sn, cs;
    const float arg = wf * th;
    sincosf(arg, &sn, &cs);
    if constexpr (kGeom) {
      // f1 = < gf, dF/dtheta >, f2 = < gf, d^2F/dtheta^2 >;  theta(u), u = c rhat_i . rhat_j:
      // d/drhat_i [ F' thetadot ] = c (f2 thetadot th_u + f1 th_uu ud) rhat_j + c f1 th_u drhat_j   (i <-> j)
      float f1 = 0.f, f2 = 0.f;
      if (is_sin) {
        f1 = gf * wf * cs;
        f2 = -gf * wf * wf * sn;
      } else if (is_cos) {
        f1 = -gf * wf * sn;
        f2 = -gf * wf * wf * cs;
      }
      f1 = sum32(f1) * inv_sqrt_pi;
      f2 = sum32(f2) * inv_sqrt_pi;
      constexpr float c = 1.f - 1e-6f;
      const float th_uu = tg.th_u * tg.th_u * tg.th_u * tg.u;  // -u / (1 - u^2)^(3/2)
      const float k_r = c * fmaf(f2 * thd, tg.th_u, f1 * th_uu * tg.ud), k_d = c * f1 * tg.th_u;
      if (lane < 3) {
        atomicAdd(g_rhat + (size_t)ang_di[a] * 3 + lane, (double)fmaf(k_r, pick3(tg.rj, lane), k_d * pick3(tg.drj, lane)));
      } else if (lane < 6) {
        const int k = lane - 3;
        atomicAdd(g_rhat + (size_t)ang_dj[a] * 3 + k, (double)fmaf(k_r, pick3(tg.ri, k), k_d * pick3(tg.dri, k)));
      }
    } else {
      // d/dw [ w cos(w th) ] = cos - w th sin ;  d/dw [ -w sin(w th) ] = -(sin + w th cos)
      if (is_sin) gfr += (double)(gf * (cs - arg * sn) * thd * inv_sqrt_pi);
      else if (is_cos) gfr -= (double)(gf * (sn + arg * cs) * thd * inv_sqrt_pi);
    }
  }
  if constexpr (!kGeom) {
    if (is_sin) atomicAdd(g_freq + lane - 1, gfr);
    else if (is_cos) atomicAdd(g_freq + lane - 1 - nf, gfr);
  }
}

// virial[graph] += sum over the block's edges of r (x) g, row i column j at [i*3 + j].  Edges are grouped by graph,
// so a block usually lies inside one graph: then a warp sum, a shared-memory sum over the 8 warps and 9 atomics per
// block.  A block that spans graphs (a batch of small cells) falls back to one atomic per edge and component.  Every
// thread of a 256-thread block calls it; threads past the last edge pass graph = -1 and r = g = 0.
__device__ __forceinline__ void block_virial_add(const double (&r)[3], const double (&g)[3], int graph,
                                                 const int32_t* __restrict__ center,
                                                 const int32_t* __restrict__ owner, int n_edges,
                                                 double* __restrict__ virial) {
  __shared__ double s_v[8][9];
  __shared__ int s_uniform;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int first = blockIdx.x * blockDim.x;
  const int last = min(first + (int)blockDim.x, n_edges) - 1;
  if (threadIdx.x == 0) s_uniform = owner[center[first]] == owner[center[last]];
  __syncthreads();
  if (s_uniform != 0) {
    double v[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) v[i * 3 + j] = sum32d(r[i] * g[j]);
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < 9; ++k) s_v[wid][k] = v[k];
    }
    __syncthreads();
    if (threadIdx.x < 9) {
      double t = 0.0;
      for (int w8 = 0; w8 < 8; ++w8) t += s_v[w8][threadIdx.x];
      atomicAdd(virial + (size_t)owner[center[first]] * 9 + threadIdx.x, t);
    }
  } else if (graph >= 0) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) atomicAdd(virial + (size_t)graph * 9 + i * 3 + j, r[i] * g[j]);
  }
}

// d/dr_e of  lam_d ddist + lam_rhat . drhat  with rdot held fixed (Hessian-vector products), scattered like
// force_virial (force[c] -= g, force[n] += g).  ddist = rhat . rdot -> drhat;  drhat = (rdot - rhat ddist)/d ->
// -[(mu . drhat) rhat + (mu . rhat) drhat + ddist (mu - rhat (rhat . mu))/d]/d,  mu = lam_rhat.  lam_d belongs to
// the bond's representative edge only (the bond basis reads d there).
// kVirial = true also adds sum_e r_e (x) g per graph to virial [B][9], as force_virial does (strain derivatives).
template <bool kVirial>
__global__ void __launch_bounds__(256)
edge_tangent_bwd_kernel(const float* __restrict__ rvec, const float* __restrict__ dist,
                        const float* __restrict__ rhat, const float* __restrict__ ddist,
                        const float* __restrict__ drhat, const float* __restrict__ lam_dist,
                        const double* __restrict__ lam_rhat, const int32_t* __restrict__ d2u,
                        const int32_t* __restrict__ u2d, const int32_t* __restrict__ center,
                        const int32_t* __restrict__ nbr, const int32_t* __restrict__ owner, int n_edges,
                        double* __restrict__ force, double* __restrict__ virial) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  double g[3] = {0.0, 0.0, 0.0}, r[3] = {0.0, 0.0, 0.0};
  int graph = -1;
  if (e < n_edges) {
    const int c = center[e], n = nbr[e], u = d2u[e];
    double rh[3], rd[3], mu[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      rh[j] = (double)rhat[(size_t)e * 3 + j];
      rd[j] = (double)drhat[(size_t)e * 3 + j];
      mu[j] = lam_rhat[(size_t)e * 3 + j];
    }
    const double inv_d = 1.0 / (double)dist[e], dd = (double)ddist[e];
    const double ld = (u2d[u] == e) ? (double)lam_dist[u] : 0.0;
    const double m_rd = mu[0] * rd[0] + mu[1] * rd[1] + mu[2] * rd[2];
    const double m_rh = mu[0] * rh[0] + mu[1] * rh[1] + mu[2] * rh[2];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      g[j] = ld * rd[j] - (m_rd * rh[j] + m_rh * rd[j] + dd * (mu[j] - rh[j] * m_rh) * inv_d) * inv_d;
      atomicAdd(force + (size_t)c * 3 + j, -g[j]);
      atomicAdd(force + (size_t)n * 3 + j, g[j]);
    }
    if constexpr (kVirial) {
      graph = owner[c];
#pragma unroll
      for (int j = 0; j < 3; ++j) r[j] = (double)rvec[(size_t)e * 3 + j];
    }
  }
  if constexpr (kVirial) block_virial_add(r, g, graph, center, owner, n_edges, virial);
}

// ---- magmom head -------------------------------------------------------------------
__global__ void magmom_kernel(const float* __restrict__ x, int n_atoms, const float* __restrict__ w, float b,
                              float* __restrict__ m) {
  const int lane = threadIdx.x & 31;
  const int atom = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (atom >= n_atoms) return;
  const float* row = x + (size_t)atom * 64;
  float v = fmaf(row[lane], w[lane], row[lane + 32] * w[lane + 32]);
  v = sum32(v);
  if (lane == 0) m[atom] = fabsf(v + b);
}

// ---- force + virial -------------------------------------------------------------------
__global__ void __launch_bounds__(256)
force_virial_kernel(const float* __restrict__ rvec, const float* __restrict__ dist, const float* __restrict__ rhat,
                    const double* __restrict__ g_rhat, const float* __restrict__ g_dist,
                    const int32_t* __restrict__ d2u, const int32_t* __restrict__ u2d,
                    const int32_t* __restrict__ center, const int32_t* __restrict__ nbr,
                    const int32_t* __restrict__ owner, int n_edges, double* __restrict__ force,
                    double* __restrict__ virial) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  double g[3] = {0.0, 0.0, 0.0}, r[3] = {0.0, 0.0, 0.0};
  int graph = -1;
  if (e < n_edges) {
    const int c = center[e], n = nbr[e], u = d2u[e];
    graph = owner[c];
    double rh[3], gr[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      rh[j] = (double)rhat[(size_t)e * 3 + j];
      gr[j] = g_rhat[(size_t)e * 3 + j];
      r[j] = (double)rvec[(size_t)e * 3 + j];
    }
    const double dot = rh[0] * gr[0] + rh[1] * gr[1] + rh[2] * gr[2];
    const double inv_d = 1.0 / (double)dist[e];
    const double gd = (u2d[u] == e) ? (double)g_dist[u] : 0.0;  // d_u is taken from its representative edge only
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      g[j] = (gr[j] - rh[j] * dot) * inv_d + gd * rh[j];
      atomicAdd(force + (size_t)c * 3 + j, -g[j]);
      atomicAdd(force + (size_t)n * 3 + j, g[j]);
    }
  }
  block_virial_add(r, g, graph, center, owner, n_edges, virial);
}

inline int warp_grid(int n_items, int threads = 256) {
  const int warps_per_block = threads / 32;
  const int need = (n_items + warps_per_block - 1) / warps_per_block;
  return max(1, min(need, sm_count() * 8));
}

}  // namespace
}  // namespace chg

using namespace chg;

extern "C" int chg_embed_atoms(const int32_t* z, const float* emb, int32_t n_atoms, float* x, void* stream) {
  CHG_CHECK_ARG(n_atoms >= 0, "negative size");
  if (n_atoms == 0) return CHG_OK;
  CHG_CHECK_ARG(z && emb && x, "null pointer");
  const int total = n_atoms * 16;
  embed_atoms_kernel<<<(total + 255) / 256, 256, 0, as_stream(stream)>>>(z, emb, n_atoms, x);
  CHG_LAUNCH_END();
}

extern "C" int chg_edge_geometry(const float* frac, const float* lattice, const int32_t* atom_owner,
                                 const int32_t* center, const int32_t* nbr, const float* image, int32_t n_edges,
                                 float* rvec, float* dist, float* rhat, void* stream) {
  CHG_CHECK_ARG(n_edges >= 0, "negative size");
  if (n_edges == 0) return CHG_OK;
  CHG_CHECK_ARG(frac && lattice && atom_owner && center && nbr && image && rvec && dist && rhat, "null pointer");
  edge_geometry_kernel<<<(n_edges + 255) / 256, 256, 0, as_stream(stream)>>>(frac, lattice, atom_owner, center, nbr,
                                                                             image, n_edges, rvec, dist, rhat);
  CHG_LAUNCH_END();
}

extern "C" int chg_bond_basis_embed(const float* dist, const int32_t* u2d, int32_t n_bonds, const float* freq_ag,
                                    const float* freq_bg, int32_t n_radial, float rc_ag, float rc_bg, int32_t p,
                                    const float* w3t, float* e0, float* wag, float* wbg, float* basis_out,
                                    void* stream) {
  CHG_CHECK_ARG(n_bonds >= 0, "negative size");
  CHG_CHECK_ARG(n_radial >= 1 && n_radial <= MAX_BASIS, "num_radial must be in [1, 32]");
  if (n_bonds == 0) return CHG_OK;
  CHG_CHECK_ARG(dist && u2d && freq_ag && freq_bg && w3t && e0 && wag && wbg, "null pointer");
  const int smem = 3 * n_radial * 64 * 4;
  bond_basis_embed_kernel<<<warp_grid((n_bonds + 3) / 4), 256, smem, as_stream(stream)>>>(
      dist, u2d, n_bonds, freq_ag, freq_bg, n_radial, rc_ag, rc_bg, p, w3t, e0, wag, wbg, basis_out);
  CHG_LAUNCH_END();
}

extern "C" int chg_bond_basis_bwd(const float* dist, const int32_t* u2d, int32_t n_bonds, const float* freq_ag,
                                  const float* freq_bg, int32_t n_radial, float rc_ag, float rc_bg, int32_t p,
                                  const float* w3, const float* g_e0, const float* g_wag, const float* g_wbg,
                                  float* g_dist, double* g_freq, void* stream) {
  CHG_CHECK_ARG(n_bonds >= 0, "negative size");
  CHG_CHECK_ARG(n_radial >= 1 && n_radial <= MAX_BASIS, "num_radial must be in [1, 32]");
  if (n_bonds == 0) return CHG_OK;
  CHG_CHECK_ARG(dist && u2d && freq_ag && freq_bg && w3 && g_e0 && g_wag && g_wbg && g_dist, "null pointer");
  const int smem = 3 * n_radial * 64 * 4;
  bond_basis_bwd_kernel<<<warp_grid((n_bonds + 1) / 2), 256, smem, as_stream(stream)>>>(
      dist, u2d, n_bonds, freq_ag, freq_bg, n_radial, rc_ag, rc_bg, p, w3, g_e0, g_wag, g_wbg, g_dist, g_freq);
  CHG_LAUNCH_END();
}

// The angle-basis entry points take freq == nullptr when n_freq == 0 (num_angular = 1: the constant term only); no
// lane reads a frequency or writes a frequency gradient then.
extern "C" int chg_angle_basis_embed(const float* rhat, const int32_t* ang_di, const int32_t* ang_dj,
                                     int32_t n_angles, const float* freq, int32_t n_freq, const float* wt, float* a0,
                                     float* basis_out, void* stream) {
  CHG_CHECK_ARG(n_angles >= 0, "negative size");
  CHG_CHECK_ARG(n_freq >= 0 && 2 * n_freq + 1 <= MAX_BASIS, "num_angular must be odd and <= 31");
  if (n_angles == 0) return CHG_OK;
  CHG_CHECK_ARG(rhat && ang_di && ang_dj && (freq || n_freq == 0) && wt && a0, "null pointer");
  const int smem = (2 * n_freq + 1) * 64 * 4;
  angle_basis_embed_kernel<<<warp_grid((n_angles + 3) / 4), 256, smem, as_stream(stream)>>>(rhat, ang_di, ang_dj, n_angles,
                                                                                  freq, n_freq, wt, a0, basis_out);
  CHG_LAUNCH_END();
}

extern "C" int chg_angle_basis_bwd(const float* rhat, const int32_t* ang_di, const int32_t* ang_dj, int32_t n_angles,
                                   const float* freq, int32_t n_freq, const float* w, const float* g_a0,
                                   double* g_rhat, double* g_freq, void* stream) {
  CHG_CHECK_ARG(n_angles >= 0, "negative size");
  CHG_CHECK_ARG(n_freq >= 0 && 2 * n_freq + 1 <= MAX_BASIS, "num_angular must be odd and <= 31");
  if (n_angles == 0 || (g_rhat == nullptr && n_freq == 0)) return CHG_OK;  // num_angular = 1: g_freq has no entries
  CHG_CHECK_ARG(rhat && ang_di && ang_dj && (freq || n_freq == 0) && w && g_a0 && (g_rhat || g_freq), "null pointer");
  const int smem = (2 * n_freq + 1) * 64 * 4;
  angle_basis_bwd_kernel<<<warp_grid((n_angles + 15) / 16), 256, smem, as_stream(stream)>>>(rhat, ang_di, ang_dj, n_angles, freq,
                                                                                n_freq, w, g_a0, g_rhat, g_freq);
  CHG_LAUNCH_END();
}

extern "C" int chg_magmom(const float* x, int32_t n_atoms, const float* w, float b, float* m, void* stream) {
  CHG_CHECK_ARG(n_atoms >= 0, "negative size");
  if (n_atoms == 0) return CHG_OK;
  CHG_CHECK_ARG(x && w && m, "null pointer");
  const int blocks = (n_atoms * 32 + 255) / 256;
  magmom_kernel<<<blocks, 256, 0, as_stream(stream)>>>(x, n_atoms, w, b, m);
  CHG_LAUNCH_END();
}

extern "C" int chg_force_virial(const float* rvec, const float* dist, const float* rhat, const double* g_rhat,
                                const float* g_dist, const int32_t* d2u, const int32_t* u2d, const int32_t* center,
                                const int32_t* nbr, const int32_t* atom_owner, int32_t n_edges, double* force,
                                double* virial, void* stream) {
  CHG_CHECK_ARG(n_edges >= 0, "negative size");
  if (n_edges == 0) return CHG_OK;
  CHG_CHECK_ARG(rvec && dist && rhat && g_rhat && g_dist && d2u && u2d && center && nbr && atom_owner && force &&
                    virial,
                "null pointer");
  force_virial_kernel<<<(n_edges + 255) / 256, 256, 0, as_stream(stream)>>>(
      rvec, dist, rhat, g_rhat, g_dist, d2u, u2d, center, nbr, atom_owner, n_edges, force, virial);
  CHG_LAUNCH_END();
}

extern "C" int chg_edge_tangent(const float* rvec, const float* dist, const float* rhat, const int32_t* center,
                                const int32_t* nbr, const int32_t* atom_owner, const float* u_atom,
                                const float* w_graph, int32_t n_edges, float* ddist, float* drhat, void* stream) {
  CHG_CHECK_ARG(n_edges >= 0, "negative size");
  if (n_edges == 0) return CHG_OK;
  CHG_CHECK_ARG(rvec && dist && rhat && center && nbr && atom_owner && u_atom && w_graph && ddist && drhat, "null pointer");
  edge_tangent_kernel<<<(n_edges + 255) / 256, 256, 0, as_stream(stream)>>>(rvec, dist, rhat, center, nbr, atom_owner,
                                                                            u_atom, w_graph, n_edges, ddist, drhat);
  CHG_LAUNCH_END();
}

extern "C" int chg_bond_basis_tangent(const float* dist, const float* ddist, const int32_t* u2d, int32_t n_bonds,
                                      const float* freq_ag, const float* freq_bg, int32_t n_radial, float rc_ag,
                                      float rc_bg, int32_t p, const float* w3t, float* e0d, float* wagd, float* wbgd,
                                      float* tbasis, void* stream) {
  CHG_CHECK_ARG(n_bonds >= 0, "negative size");
  CHG_CHECK_ARG(n_radial >= 1 && n_radial <= MAX_BASIS, "num_radial must be in [1, 32]");
  if (n_bonds == 0) return CHG_OK;
  CHG_CHECK_ARG(dist && ddist && u2d && freq_ag && freq_bg && w3t && e0d && wagd && wbgd && tbasis, "null pointer");
  const int smem = 3 * n_radial * 64 * 4;
  bond_basis_tangent_kernel<<<warp_grid(n_bonds), 256, smem, as_stream(stream)>>>(
      dist, ddist, u2d, n_bonds, freq_ag, freq_bg, n_radial, rc_ag, rc_bg, p, w3t, e0d, wagd, wbgd, tbasis);
  CHG_LAUNCH_END();
}

extern "C" int chg_bond_basis_bwd2(const float* dist, const float* ddist, const int32_t* u2d, int32_t n_bonds,
                                   const float* freq_ag, const float* freq_bg, int32_t n_radial, float rc_ag,
                                   float rc_bg, int32_t p, const float* w3, const float* lam_e0, const float* lam_wag,
                                   const float* lam_wbg, double* g_freq, void* stream) {
  CHG_CHECK_ARG(n_bonds >= 0, "negative size");
  CHG_CHECK_ARG(n_radial >= 1 && n_radial <= MAX_BASIS, "num_radial must be in [1, 32]");
  if (n_bonds == 0) return CHG_OK;
  CHG_CHECK_ARG(dist && ddist && u2d && freq_ag && freq_bg && w3 && lam_e0 && lam_wag && lam_wbg && g_freq, "null pointer");
  const int smem = 3 * n_radial * 64 * 4;
  bond_basis_bwd2_kernel<false><<<warp_grid(n_bonds), 256, smem, as_stream(stream)>>>(
      dist, ddist, u2d, n_bonds, freq_ag, freq_bg, n_radial, rc_ag, rc_bg, p, w3, lam_e0, lam_wag, lam_wbg, g_freq,
      nullptr);
  CHG_LAUNCH_END();
}

extern "C" int chg_bond_basis_hvp(const float* dist, const float* ddist, const int32_t* u2d, int32_t n_bonds,
                                  const float* freq_ag, const float* freq_bg, int32_t n_radial, float rc_ag,
                                  float rc_bg, int32_t p, const float* w3, const float* lam_e0, const float* lam_wag,
                                  const float* lam_wbg, float* g_dist, void* stream) {
  CHG_CHECK_ARG(n_bonds >= 0, "negative size");
  CHG_CHECK_ARG(n_radial >= 1 && n_radial <= MAX_BASIS, "num_radial must be in [1, 32]");
  if (n_bonds == 0) return CHG_OK;
  CHG_CHECK_ARG(dist && ddist && u2d && freq_ag && freq_bg && w3 && lam_e0 && lam_wag && lam_wbg && g_dist, "null pointer");
  const int smem = 3 * n_radial * 64 * 4;
  bond_basis_bwd2_kernel<true><<<warp_grid(n_bonds), 256, smem, as_stream(stream)>>>(
      dist, ddist, u2d, n_bonds, freq_ag, freq_bg, n_radial, rc_ag, rc_bg, p, w3, lam_e0, lam_wag, lam_wbg, nullptr,
      g_dist);
  CHG_LAUNCH_END();
}

extern "C" int chg_angle_basis_tangent(const float* rhat, const float* drhat, const int32_t* ang_di,
                                       const int32_t* ang_dj, int32_t n_angles, const float* freq, int32_t n_freq,
                                       const float* wt, float* a0d, float* tbasis, void* stream) {
  CHG_CHECK_ARG(n_angles >= 0, "negative size");
  CHG_CHECK_ARG(n_freq >= 0 && 2 * n_freq + 1 <= MAX_BASIS, "num_angular must be odd and <= 31");
  if (n_angles == 0) return CHG_OK;
  CHG_CHECK_ARG(rhat && drhat && ang_di && ang_dj && (freq || n_freq == 0) && wt && a0d && tbasis, "null pointer");
  const int smem = (2 * n_freq + 1) * 64 * 4;
  angle_basis_tangent_kernel<<<warp_grid(n_angles), 256, smem, as_stream(stream)>>>(rhat, drhat, ang_di, ang_dj, n_angles,
                                                                                   freq, n_freq, wt, a0d, tbasis);
  CHG_LAUNCH_END();
}

extern "C" int chg_angle_basis_bwd2(const float* rhat, const float* drhat, const int32_t* ang_di, const int32_t* ang_dj,
                                    int32_t n_angles, const float* freq, int32_t n_freq, const float* w,
                                    const float* lam_a0, double* g_freq, void* stream) {
  CHG_CHECK_ARG(n_angles >= 0, "negative size");
  CHG_CHECK_ARG(n_freq >= 0 && 2 * n_freq + 1 <= MAX_BASIS, "num_angular must be odd and <= 31");
  if (n_angles == 0 || n_freq == 0) return CHG_OK;  // num_angular = 1: g_freq has no entries
  CHG_CHECK_ARG(rhat && drhat && ang_di && ang_dj && (freq || n_freq == 0) && w && lam_a0 && g_freq, "null pointer");
  const int smem = (2 * n_freq + 1) * 64 * 4;
  angle_basis_bwd2_kernel<false><<<warp_grid(n_angles), 256, smem, as_stream(stream)>>>(
      rhat, drhat, ang_di, ang_dj, n_angles, freq, n_freq, w, lam_a0, g_freq, nullptr);
  CHG_LAUNCH_END();
}

extern "C" int chg_angle_basis_hvp(const float* rhat, const float* drhat, const int32_t* ang_di, const int32_t* ang_dj,
                                   int32_t n_angles, const float* freq, int32_t n_freq, const float* w,
                                   const float* lam_a0, double* g_rhat, void* stream) {
  CHG_CHECK_ARG(n_angles >= 0, "negative size");
  CHG_CHECK_ARG(n_freq >= 0 && 2 * n_freq + 1 <= MAX_BASIS, "num_angular must be odd and <= 31");
  if (n_angles == 0) return CHG_OK;
  CHG_CHECK_ARG(rhat && drhat && ang_di && ang_dj && (freq || n_freq == 0) && w && lam_a0 && g_rhat, "null pointer");
  const int smem = (2 * n_freq + 1) * 64 * 4;
  angle_basis_bwd2_kernel<true><<<warp_grid(n_angles), 256, smem, as_stream(stream)>>>(
      rhat, drhat, ang_di, ang_dj, n_angles, freq, n_freq, w, lam_a0, nullptr, g_rhat);
  CHG_LAUNCH_END();
}

extern "C" int chg_edge_tangent_bwd(const float* dist, const float* rhat, const float* ddist, const float* drhat,
                                    const float* lam_dist, const double* lam_rhat, const int32_t* d2u,
                                    const int32_t* u2d, const int32_t* center, const int32_t* nbr, int32_t n_edges,
                                    double* force, void* stream) {
  CHG_CHECK_ARG(n_edges >= 0, "negative size");
  if (n_edges == 0) return CHG_OK;
  CHG_CHECK_ARG(dist && rhat && ddist && drhat && lam_dist && lam_rhat && d2u && u2d && center && nbr && force,
                "null pointer");
  edge_tangent_bwd_kernel<false><<<(n_edges + 255) / 256, 256, 0, as_stream(stream)>>>(
      nullptr, dist, rhat, ddist, drhat, lam_dist, lam_rhat, d2u, u2d, center, nbr, nullptr, n_edges, force, nullptr);
  CHG_LAUNCH_END();
}

extern "C" int chg_edge_tangent_bwd_virial(const float* rvec, const float* dist, const float* rhat,
                                           const float* ddist, const float* drhat, const float* lam_dist,
                                           const double* lam_rhat, const int32_t* d2u, const int32_t* u2d,
                                           const int32_t* center, const int32_t* nbr, const int32_t* atom_owner,
                                           int32_t n_edges, double* force, double* virial, void* stream) {
  CHG_CHECK_ARG(n_edges >= 0, "negative size");
  if (n_edges == 0) return CHG_OK;
  CHG_CHECK_ARG(rvec && dist && rhat && ddist && drhat && lam_dist && lam_rhat && d2u && u2d && center && nbr &&
                    atom_owner && force && virial,
                "null pointer");
  edge_tangent_bwd_kernel<true><<<(n_edges + 255) / 256, 256, 0, as_stream(stream)>>>(
      rvec, dist, rhat, ddist, drhat, lam_dist, lam_rhat, d2u, u2d, center, nbr, atom_owner, n_edges, force, virial);
  CHG_LAUNCH_END();
}
