// Device-resident molecular dynamics / relaxation updates (SURVEY.md §8 row f2).
//
// The reference keeps positions in an ase.Atoms object on the host and calls the model once per step through
// CHGNetCalculator.calculate (chgnet/model/dynamics.py:129-181): structure -> graph on the CPU -> H2D -> model -> D2H.
// Here positions, velocities and forces stay on the device in fp64; these kernels are the integrator halves that sit
// on either side of chg_forward inside ONE CUDA graph per step (chgnet_b200/dynamics_device.py):
//   chg_md_kick_drift : v += dt/2 F/m ; x += dt v ; frac = x L^-1 (fp64 for the graph builder, fp32 for the model);
//                       max |x - x_ref|^2 for the neighbour-list skin test
//   chg_md_kick       : v += dt/2 F/m ; kinetic energy
//   chg_fire_step     : FIRE (Bitzek et al. 2006; the reference's default optimizer, dynamics.py:190-204) with its
//                       state (dt, alpha, counters) in device memory: four launches, no host decision in the loop
#include "common.cuh"

namespace chg {
namespace {

struct Mat3 {
  double m[9];
};

__device__ __forceinline__ void atomic_max_nonneg(double* addr, double v) {
  // non-negative doubles order like their bit patterns
  atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)__double_as_longlong(v));
}

__global__ void md_kick_drift_kernel(double* __restrict__ x, double* __restrict__ v, const double* __restrict__ f,
                                     const double* __restrict__ inv_mass, int n, double dt, Mat3 inv_l,
                                     double* __restrict__ frac64, float* __restrict__ frac32, const double* __restrict__ x_ref,
                                     double* __restrict__ max_disp2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double im = inv_mass[i];
  double xi[3], d2 = 0.0;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const double vj = v[3 * i + j] + 0.5 * dt * f[3 * i + j] * im;
    v[3 * i + j] = vj;
    xi[j] = x[3 * i + j] + dt * vj;
    x[3 * i + j] = xi[j];
    if (x_ref != nullptr) {
      const double d = xi[j] - x_ref[3 * i + j];
      d2 += d * d;
    }
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const double fj = xi[0] * inv_l.m[j] + xi[1] * inv_l.m[3 + j] + xi[2] * inv_l.m[6 + j];
    frac64[3 * i + j] = fj;
    frac32[3 * i + j] = (float)fj;
  }
  if (max_disp2 != nullptr) atomic_max_nonneg(max_disp2, d2);
}

__global__ void md_kick_kernel(double* __restrict__ v, const double* __restrict__ f, const double* __restrict__ inv_mass, int n,
                               double dt, double* __restrict__ e_kin) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double ke = 0.0;
  if (i < n) {
    const double im = inv_mass[i];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double vj = v[3 * i + j] + 0.5 * dt * f[3 * i + j] * im;
      v[3 * i + j] = vj;
      ke += vj * vj;
    }
    ke *= 0.5 / im;
  }
  ke = sum32d(ke);
  if (e_kin != nullptr && (threadIdx.x & 31) == 0 && ke != 0.0) atomicAdd(e_kin, ke);
}

// FIRE state in device memory (the 12 slots are documented at chg_fire_step in include/chgnet_b200.h): [0] dt, [1] alpha,
// [2] n_pos (as double); scratch [3] power, [4] |v|^2, [5] |f|^2, [6] max |f_i|^2, [7] max |dt v_i|^2 of this update;
// published [8..10] the new dt, alpha, n_pos and [11] max |f_i|^2
__global__ void fire_reduce_kernel(const double* __restrict__ v, const double* __restrict__ f, int n, double* __restrict__ st) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double p = 0.0, vv = 0.0, ff = 0.0;
  if (i < n) {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double vj = v[3 * i + j], fj = f[3 * i + j];
      p += fj * vj;
      vv += vj * vj;
      ff += fj * fj;
    }
    atomic_max_nonneg(st + 6, ff);
  }
  p = sum32d(p);
  vv = sum32d(vv);
  ff = sum32d(ff);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(st + 3, p);
    atomicAdd(st + 4, vv);
    atomicAdd(st + 5, ff);
  }
}

__global__ void fire_update_kernel(double* __restrict__ v, const double* __restrict__ f, int n, double* __restrict__ st,
                                   double dt_max) {
  // every thread derives the same scalars from the reduced state (written by the previous launch)
  const double n_min = 5.0, f_inc = 1.1, f_dec = 0.5, alpha_start = 0.1, f_alpha = 0.99;
  double dt = st[0], alpha = st[1], n_pos = st[2];
  const double power = st[3], vnorm = sqrt(st[4]), fnorm = sqrt(st[5]);
  const bool uphill = !(power > 0.0);
  if (!uphill) {
    n_pos += 1.0;
    if (n_pos > n_min) {
      dt = fmin(dt * f_inc, dt_max);
      alpha *= f_alpha;
    }
  } else {
    dt *= f_dec;
    alpha = alpha_start;
    n_pos = 0.0;
  }
  const double mix = uphill ? 0.0 : st[1] * vnorm / fmax(fnorm, 1e-30);
  const double keep = uphill ? 0.0 : 1.0 - st[1];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    double d2 = 0.0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double vn = keep * v[3 * i + j] + mix * f[3 * i + j] + dt * f[3 * i + j];
      const double dr = dt * vn;
      v[3 * i + j] = vn;
      d2 += dr * dr;
    }
    // no atom moves yet: the step limit needs the largest per-atom step of the whole update (fire_move)
    atomic_max_nonneg(st + 7, d2);
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    // the new scalars for fire_move, the host and the next step
    st[8] = dt;
    st[9] = alpha;
    st[10] = n_pos;
    st[11] = st[6];  // max |f_i|^2 seen by this step
  }
}

// x += s dt v with one scale s = min(1, max_step / max_i |dt v_i|) for all atoms (fire_relax's step limit: the update
// keeps its direction, every atom keeps its share of it); v itself is not scaled
__global__ void fire_move_kernel(double* __restrict__ x, const double* __restrict__ v, int n, const double* __restrict__ st,
                                 Mat3 inv_l, double* __restrict__ frac64, float* __restrict__ frac32, double max_step) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double dt = st[8], norm = sqrt(st[7]);
  const double s = norm > max_step ? max_step / norm : 1.0;
  double xi[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    xi[j] = x[3 * i + j] + (dt * v[3 * i + j]) * s;
    x[3 * i + j] = xi[j];
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const double fj = xi[0] * inv_l.m[j] + xi[1] * inv_l.m[3 + j] + xi[2] * inv_l.m[6 + j];
    frac64[3 * i + j] = fj;
    frac32[3 * i + j] = (float)fj;
  }
}

// commits the scalars of fire_update (a separate tiny launch: every block of the update must have read the old ones)
__global__ void fire_commit_kernel(double* __restrict__ st) {
  st[0] = st[8];
  st[1] = st[9];
  st[2] = st[10];
  st[3] = st[4] = st[5] = st[6] = st[7] = 0.0;
}

inline unsigned blocks(int n) { return (unsigned)((n + 255) / 256); }

}  // namespace
}  // namespace chg

using namespace chg;

extern "C" int chg_md_kick_drift(double* x, double* v, const double* f, const double* inv_mass, int32_t n_atoms, double dt,
                                 const double* inv_lattice /* host, 9 */, double* frac64, float* frac32, const double* x_ref,
                                 double* max_disp2, void* stream) {
  CHG_CHECK_ARG(n_atoms >= 0, "negative size");
  if (n_atoms == 0) return CHG_OK;
  CHG_CHECK_ARG(x && v && f && inv_mass && inv_lattice && frac64 && frac32, "null pointer");
  Mat3 il;
  for (int i = 0; i < 9; ++i) il.m[i] = inv_lattice[i];
  md_kick_drift_kernel<<<blocks(n_atoms), 256, 0, as_stream(stream)>>>(x, v, f, inv_mass, n_atoms, dt, il, frac64, frac32, x_ref, max_disp2);
  CHG_LAUNCH_END();
}

extern "C" int chg_md_kick(double* v, const double* f, const double* inv_mass, int32_t n_atoms, double dt, double* e_kin,
                           void* stream) {
  CHG_CHECK_ARG(n_atoms >= 0, "negative size");
  if (n_atoms == 0) return CHG_OK;
  CHG_CHECK_ARG(v && f && inv_mass, "null pointer");
  md_kick_kernel<<<blocks(n_atoms), 256, 0, as_stream(stream)>>>(v, f, inv_mass, n_atoms, dt, e_kin);
  CHG_LAUNCH_END();
}

extern "C" int chg_fire_step(double* x, double* v, const double* f, int32_t n_atoms, double* state /* device, 12 doubles */,
                             const double* inv_lattice /* host, 9 */, double* frac64, float* frac32, double dt_max,
                             double max_step, void* stream) {
  CHG_CHECK_ARG(n_atoms >= 0, "negative size");
  if (n_atoms == 0) return CHG_OK;
  CHG_CHECK_ARG(x && v && f && state && inv_lattice && frac64 && frac32, "null pointer");
  Mat3 il;
  for (int i = 0; i < 9; ++i) il.m[i] = inv_lattice[i];
  cudaStream_t st = as_stream(stream);
  fire_reduce_kernel<<<blocks(n_atoms), 256, 0, st>>>(v, f, n_atoms, state);
  count_launch();
  fire_update_kernel<<<blocks(n_atoms), 256, 0, st>>>(v, f, n_atoms, state, dt_max);
  count_launch();
  fire_move_kernel<<<blocks(n_atoms), 256, 0, st>>>(x, v, n_atoms, state, il, frac64, frac32, max_step);
  count_launch();
  fire_commit_kernel<<<1, 1, 0, st>>>(state);
  CHG_LAUNCH_END();
}
