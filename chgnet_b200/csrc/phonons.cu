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
//
// The same sum with every image term multiplied by 2 pi i r_c, r = v . prim_lattice the Cartesian image vector (A), is
// dD/dQ_c, the derivative with respect to the Cartesian wave vector Q = q . inv(prim_lattice)^T (no 2 pi; q.v = Q.r):
// the group velocities of Phonons.group_velocities.  One more grid dimension runs over c.
//
// chg_tetrahedron_dos: the linear tetrahedron method (Bloechl's closed forms) on a full Gamma-centred mesh, see below.
// chg_thermal_displacements: the mode- and temperature-weighted sums of Re(e e^H) per atom behind the thermal
// displacement matrices, see below.
// chg_joint_dos: the two-phonon joint densities of states D2 and their occupation-weighted forms N2 at target q-points,
// by the same tetrahedron method, see below.
// chg_structure_factors and chg_broadened_spectrum: coherent one-phonon neutron structure factors S(Q, omega) per mode
// and their Gaussian-broadened spectra, averaged over groups of rows (powder directions), see below.
#include <math_constants.h>

#include <algorithm>

#include "common.cuh"

namespace chg {
namespace {

constexpr int DYN_THREADS = 128;  // q-points per block

// re / im [3][3] = sum_{j : s2p[j] = kp} Phi[k, j] (1/m) sum_images e^{2 pi i q.v}, times 2 pi i r_c per image with
// DERIV (r_c = v . (l0, l1, l2), the column c of the primitive lattice)
template <bool DERIV>
__device__ __forceinline__ void phase_block(const double* __restrict__ fc, const int32_t* __restrict__ img_ptr,
                                            const double* __restrict__ img_vec, const int32_t* __restrict__ s2p,
                                            int n_super, int k, int kp, double q0, double q1, double q2,
                                            double l0, double l1, double l2, double (&re)[9], double (&im)[9]) {
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
      if constexpr (DERIV) {
        const double r = fma(__ldg(v), l0, fma(__ldg(v + 1), l1, __ldg(v + 2) * l2));
        c = fma(-r, sn, c);  // Re(i r e^{i phi})
        s = fma(r, cs, s);
      } else {
        c += cs;
        s += sn;
      }
    }
    double inv_m;
    if constexpr (DERIV) {
      inv_m = 6.283185307179586 / (double)(e - b);  // 2 pi
    } else {
      inv_m = 1.0 / (double)(e - b);
    }
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

// D(q) [n_q][3n][3n], or with DERIV dD/dQ_c [n_q][3][3n][3n] (c = blockIdx.z, lattice the primitive lattice [3][3])
template <bool DERIV>
__global__ void __launch_bounds__(DYN_THREADS)
dynamical_matrices_kernel(const double* __restrict__ fc, const int32_t* __restrict__ img_ptr,
                          const double* __restrict__ img_vec, const int32_t* __restrict__ s2p,
                          const double* __restrict__ inv_sqrt_m, int n_prim, int n_super,
                          const double* __restrict__ qpoints, int n_q, const double* __restrict__ lattice,
                          double* __restrict__ dyn) {
  const int k = blockIdx.x / n_prim, kp = blockIdx.x % n_prim;
  if (kp < k) return;  // block (kp, k) writes this pair
  const int iq = blockIdx.y * DYN_THREADS + threadIdx.x;
  if (iq >= n_q) return;
  const double q0 = qpoints[iq * 3], q1 = qpoints[iq * 3 + 1], q2 = qpoints[iq * 3 + 2];
  double l0 = 0.0, l1 = 0.0, l2 = 0.0;
  if constexpr (DERIV) {
    const int c = blockIdx.z;
    l0 = lattice[c], l1 = lattice[3 + c], l2 = lattice[6 + c];
  }
  double r1[9], i1[9], r2[9], i2[9];
  phase_block<DERIV>(fc, img_ptr, img_vec, s2p, n_super, k, kp, q0, q1, q2, l0, l1, l2, r1, i1);
  if (kp != k) {
    phase_block<DERIV>(fc, img_ptr, img_vec, s2p, n_super, kp, k, q0, q1, q2, l0, l1, l2, r2, i2);
  } else {
#pragma unroll
    for (int i = 0; i < 9; ++i) r2[i] = r1[i], i2[i] = i1[i];
  }
  const double w = 0.5 * inv_sqrt_m[k] * inv_sqrt_m[kp];
  const size_t n3 = 3 * (size_t)n_prim;
  const size_t mat = DERIV ? (size_t)iq * 3 + blockIdx.z : (size_t)iq;
  double* dq = dyn + mat * n3 * n3 * 2;
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

// ---------------------------------------------------------------------------------------------------------------
// Linear tetrahedron method.  Mesh cell (i, j, k) of the Gamma-centred mesh (q index (i n2 + j) n3 + k) is cut into 6
// tetrahedra given by corner offsets tet[6][4][3] in {0, 1} (periodic wrap); each band is interpolated linearly on
// each tetrahedron.  For sorted vertex values e0 <= e1 <= e2 <= e3 and the interpolant e(x), per unit volume:
//   n(w) = vol{e <= w},  g(w) = dn/dw = int delta(w - e),  wt_i(w) = int delta(w - e) lambda_i  (sum_i wt_i = g),
// lambda_i the barycentric coordinates.  The cross-section e = w is a triangle (w < e1, w >= e2) or a quadrilateral;
// wt_i / g is the lambda_i of its centroid.  With f_ij = (w - e_j) / (e_i - e_j):
//   e0 <= w < e1:  n = f10 f20 f30,  g = 3 f10 f20 / e30,  wt_j = g f_j0 / 3 (j > 0)
//   e1 <= w < e2:  n (Bloechl) = [e10^2 + 3 e10 x + 3 x^2 - (e20 + e31) x^3 / (e21 e31)] / (e20 e30), x = w - e1;
//                  g = 3 (f12 f20 + f21 f13) / e30.  The diagonal f02-f13 cuts the quadrilateral into triangles whose
//                  areas are g (1 - s) and g s, g s = 3 f13 f20 / e30, so wt_0 = (g f02 + gs f03) / 3,
//                  wt_1 = (g f13 + (g - gs) f12) / 3, wt_2 = (g f20 + (g - gs) f21) / 3, wt_3 = (g f31 + gs f30) / 3
//   e2 <= w < e3:  n = 1 - f03 f13 f23,  g = 3 f03 f13 / e32,  wt_i = g f_i3 / 3 (i < 3)
// and in each triangle case the remaining vertex takes g - the others.  The half-open intervals keep every divisor
// non-zero, whatever values coincide.
constexpr int DOS_MAX_THREADS = 256;  // frequency points per block, and pairs staged per tile
constexpr int DOS_PROJ = 4;           // projection columns per block (grid z)

__device__ __forceinline__ bool tetra_weights(double w, const double (&e)[4], double& n, double& g, double (&wt)[4]) {
  if (w >= e[3]) {
    n = 1.0;
    return false;
  }
  if (w < e[1]) {
    const double f10 = (w - e[0]) / (e[1] - e[0]), f20 = (w - e[0]) / (e[2] - e[0]), f30 = (w - e[0]) / (e[3] - e[0]);
    n = f10 * f20 * f30;
    g = 3.0 * f10 * f20 / (e[3] - e[0]);
    const double g3 = g * (1.0 / 3.0);
    wt[1] = g3 * f10, wt[2] = g3 * f20, wt[3] = g3 * f30;
    wt[0] = g - wt[1] - wt[2] - wt[3];
  } else if (w < e[2]) {
    const double e10 = e[1] - e[0], e20 = e[2] - e[0], e30 = e[3] - e[0], e21 = e[2] - e[1], e31 = e[3] - e[1];
    const double x = w - e[1];
    n = (e10 * e10 + 3.0 * e10 * x + 3.0 * x * x - (e20 + e31) * x * x * x / (e21 * e31)) / (e20 * e30);
    const double f02 = (w - e[2]) / (e[0] - e[2]), f03 = (w - e[3]) / (e[0] - e[3]);
    const double f12 = (w - e[2]) / (e[1] - e[2]), f13 = (w - e[3]) / (e[1] - e[3]);
    const double f20 = 1.0 - f02, f30 = 1.0 - f03, f21 = 1.0 - f12, f31 = 1.0 - f13;
    g = 3.0 * (f12 * f20 + f21 * f13) / e30;
    const double gs = 3.0 * f13 * f20 / e30, gr = g - gs;
    wt[0] = (g * f02 + gs * f03) * (1.0 / 3.0);
    wt[1] = (g * f13 + gr * f12) * (1.0 / 3.0);
    wt[2] = (g * f20 + gr * f21) * (1.0 / 3.0);
    wt[3] = (g * f31 + gs * f30) * (1.0 / 3.0);
  } else {
    const double f03 = (e[3] - w) / (e[3] - e[0]), f13 = (e[3] - w) / (e[3] - e[1]), f23 = (e[3] - w) / (e[3] - e[2]);
    n = 1.0 - f03 * f13 * f23;
    g = 3.0 * f03 * f13 / (e[3] - e[2]);
    const double g3 = g * (1.0 / 3.0);
    wt[0] = g3 * f03, wt[1] = g3 * f13, wt[2] = g3 * f23;
    wt[3] = g - wt[0] - wt[1] - wt[2];
  }
  return true;
}

// corner(v, a, b, c) for the four corners v of tetrahedron tt % 6 of mesh cell tt / 6, (a, b, c) wrapped onto the mesh
template <class Corner>
__device__ __forceinline__ void tetrahedron_corners(const int32_t* __restrict__ tet, int64_t tt, int n1, int n2, int n3,
                                                    Corner corner) {
  const int it = (int)(tt % 6);
  const int64_t cell = tt / 6;
  const int ci = (int)(cell / ((int64_t)n2 * n3)), cj = (int)((cell / n3) % n2), ck = (int)(cell % n3);
#pragma unroll
  for (int v = 0; v < 4; ++v) {
    const int32_t* o = tet + (it * 4 + v) * 3;
    int a = ci + __ldg(o), b = cj + __ldg(o + 1), c = ck + __ldg(o + 2);
    a -= a >= n1 ? n1 : 0;
    b -= b >= n2 ? n2 : 0;
    c -= c >= n3 ? n3 : 0;
    corner(v, a, b, c);
  }
}

// Sorting network: the corner values ascending, each carrying its payload (ties keep a fixed, data-determined order)
template <class T>
__device__ __forceinline__ void sort4(double (&e)[4], T (&x)[4]) {
  const auto cswap = [&](int i, int j) {
    if (e[j] < e[i]) {
      const double te = e[i];
      e[i] = e[j], e[j] = te;
      const T tx = x[i];
      x[i] = x[j], x[j] = tx;
    }
  };
  cswap(0, 1), cswap(2, 3), cswap(0, 2), cswap(1, 3), cswap(1, 2);
}

// One thread per frequency point; block x owns a contiguous range of (tetrahedron, band) pairs, z a group of
// DOS_PROJ projection columns.  Each tile of pairs is staged, sorted, in shared memory by the block and then read
// by every thread (broadcasts).  The block's sums go to work[chunk][row][F] (row 0 g, 1 n, 2 + s the projection s),
// each element written by exactly one thread: no atomics, and chunk_reduce_kernel adds the chunks in a fixed order.
__global__ void __launch_bounds__(DOS_MAX_THREADS)
tetrahedron_dos_kernel(const double* __restrict__ freqs, int n_band, int n1, int n2, int n3,
                       const int32_t* __restrict__ tet, const double* __restrict__ proj, int n_proj,
                       const double* __restrict__ omega, int n_freq, int64_t n_pairs, double* __restrict__ work) {
  __shared__ double se[DOS_MAX_THREADS][4];
  __shared__ int32_t sq[DOS_MAX_THREADS][4];
  __shared__ int32_t sb[DOS_MAX_THREADS];
  const int f = blockIdx.y * blockDim.x + threadIdx.x;
  const bool active = f < n_freq;
  const double w = active ? omega[f] : 0.0;
  const int s0 = blockIdx.z * DOS_PROJ;
  const int ns = proj ? min(DOS_PROJ, n_proj - s0) : 0;
  double acc_g = 0.0, acc_n = 0.0, acc_p[DOS_PROJ];
#pragma unroll
  for (int s = 0; s < DOS_PROJ; ++s) acc_p[s] = 0.0;
  const int64_t tile = blockDim.x;
  const int64_t n_tiles = (n_pairs + tile - 1) / tile;
  const int64_t t_end = n_tiles * (blockIdx.x + 1) / gridDim.x;
  for (int64_t t = n_tiles * blockIdx.x / gridDim.x; t < t_end; ++t) {
    const int64_t p = t * tile + threadIdx.x;
    __syncthreads();  // the previous tile has been read
    if (p < n_pairs) {
      const int band = (int)(p % n_band);
      double e[4];
      int32_t q[4];
      tetrahedron_corners(tet, p / n_band, n1, n2, n3, [&](int v, int a, int b, int c) {
        q[v] = (a * n2 + b) * n3 + c;
        e[v] = __ldg(freqs + (int64_t)q[v] * n_band + band);
      });
      sort4(e, q);
#pragma unroll
      for (int v = 0; v < 4; ++v) se[threadIdx.x][v] = e[v], sq[threadIdx.x][v] = q[v];
      sb[threadIdx.x] = band;
    }
    __syncthreads();
    if (!active) continue;
    const int n_here = (int)min(tile, n_pairs - t * tile);
    for (int i = 0; i < n_here; ++i) {
      const double e[4] = {se[i][0], se[i][1], se[i][2], se[i][3]};
      if (w < e[0]) continue;
      double n, g, wt[4];
      const bool inside = tetra_weights(w, e, n, g, wt);
      acc_n += n;
      if (!inside) continue;
      acc_g += g;
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const double* pv = proj + ((int64_t)sq[i][v] * n_band + sb[i]) * n_proj + s0;
#pragma unroll
        for (int s = 0; s < DOS_PROJ; ++s)
          if (s < ns) acc_p[s] = fma(wt[v], __ldg(pv + s), acc_p[s]);
      }
    }
  }
  if (!active) return;
  const int rows = 2 + (proj ? n_proj : 0);
  double* out = work + (size_t)blockIdx.x * rows * n_freq + f;
  if (blockIdx.z == 0) {
    out[0] = acc_g;
    out[n_freq] = acc_n;
  }
#pragma unroll
  for (int s = 0; s < DOS_PROJ; ++s)
    if (s < ns) out[(size_t)(2 + s0 + s) * n_freq] = acc_p[s];
}

struct DosStore {  // work[chunk][row][f]: scale * the sum, row 0 to dos, 1 to idos, 2 + s to pdos[s]
  double *dos, *idos, *pdos;
  int n_freq;
  double scale;
  __device__ void operator()(int64_t o, double s) const {
    const int r = (int)(o / n_freq), f = (int)(o % n_freq);
    double* out = r == 0 ? dos : (r == 1 ? idos : pdos + (size_t)(r - 2) * n_freq);
    out[f] = s * scale;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// Thermal displacements.  acc[t][k][c] += sum over (q, mode) of w(nu, T_t) Re(e e^H)_c, e the 3-component block of
// atom k in the mode's unit eigenvector, c in Voigt order (xx, yy, zz, yz, xz, xy), and
//   w = (1 + 2 / expm1(h nu / k T)) / nu  for nu >= cutoff,  0 otherwise  (1 + 2n = 1 at T = 0).
// Grid x: contiguous ranges of q (chunks); y: groups of TD_ATOMS atoms; z: tiles of temperatures.  Thread (qi, ti)
// takes the q-points q_begin + qi, q_begin + qi + n_qi, ... of its block's range at temperature t0 + ti, reads the
// eigenvector blocks of the group's atoms (the same addresses for every ti of one q) and keeps 6 TD_ATOMS sums in
// registers.  The block adds them over qi in a fixed order in shared memory and writes work[chunk][t][k][6];
// chunk_reduce_kernel adds the chunks in chunk order to acc.  No atomics, and neither the (q, mode) products nor the
// weights ever reach global memory.
constexpr int TD_THREADS = 256;  // (q, temperature) slots per block
constexpr int TD_ATOMS = 4;      // atoms per block (grid y)
// h / k_B in K/THz: chgnet_b200.phonons.H_EV_PER_THZ / chgnet_b200.dynamics.KB, the same expression in the same order
constexpr double TD_H_OVER_K = 6.62607015e-34 / 1.602176634e-19 * 1e12 / 8.617333262e-5;

__global__ void __launch_bounds__(TD_THREADS)
thermal_displacements_kernel(const double* __restrict__ freqs, const double2* __restrict__ eigvecs, int n_q,
                             int n_prim, const double* __restrict__ temps, int n_t, int t_tile, double cutoff,
                             double* __restrict__ work) {
  __shared__ double red[TD_THREADS * 6];
  const int n3 = 3 * n_prim;
  const int n_qi = blockDim.x / t_tile;  // q-points per pass
  const int qi = threadIdx.x / t_tile, ti = threadIdx.x % t_tile;
  const int t0 = blockIdx.z * t_tile, k0 = blockIdx.y * TD_ATOMS;
  const int n_here = min(TD_ATOMS, n_prim - k0);
  const bool active = t0 + ti < n_t;
  const double temp = active ? temps[t0 + ti] : 0.0;
  const int q_begin = (int)((int64_t)n_q * blockIdx.x / gridDim.x);
  const int q_end = (int)((int64_t)n_q * (blockIdx.x + 1) / gridDim.x);
  double acc[TD_ATOMS][6];
#pragma unroll
  for (int a = 0; a < TD_ATOMS; ++a)
#pragma unroll
    for (int c = 0; c < 6; ++c) acc[a][c] = 0.0;
  for (int q = q_begin + qi; active && q < q_end; q += n_qi) {
    const double* nu_q = freqs + (size_t)q * n3;
    const double2* e_q = eigvecs + (size_t)q * n3 * n3 + 3 * k0;
    for (int m = 0; m < n3; ++m) {
      const double nu = __ldg(nu_q + m);
      if (!(nu >= cutoff)) continue;
      const double coth = temp > 0.0 ? 1.0 + 2.0 / expm1(TD_H_OVER_K * nu / temp) : 1.0;
      const double w = coth / nu;
      const double2* e = e_q + (size_t)m * n3;
#pragma unroll
      for (int a = 0; a < TD_ATOMS; ++a) {
        if (a >= n_here) break;
        const double2 x = __ldg(e + 3 * a), y = __ldg(e + 3 * a + 1), z = __ldg(e + 3 * a + 2);
        acc[a][0] = fma(w, fma(x.x, x.x, x.y * x.y), acc[a][0]);
        acc[a][1] = fma(w, fma(y.x, y.x, y.y * y.y), acc[a][1]);
        acc[a][2] = fma(w, fma(z.x, z.x, z.y * z.y), acc[a][2]);
        acc[a][3] = fma(w, fma(y.x, z.x, y.y * z.y), acc[a][3]);
        acc[a][4] = fma(w, fma(x.x, z.x, x.y * z.y), acc[a][4]);
        acc[a][5] = fma(w, fma(x.x, y.x, x.y * y.y), acc[a][5]);
      }
    }
  }
  const int n_out = min(t_tile, n_t - t0) * 6;
#pragma unroll
  for (int a = 0; a < TD_ATOMS; ++a) {
    if (a >= n_here) break;  // uniform across the block
    __syncthreads();  // the previous atom's sums have been read
#pragma unroll
    for (int c = 0; c < 6; ++c) red[threadIdx.x * 6 + c] = acc[a][c];
    __syncthreads();
    for (int o = threadIdx.x; o < n_out; o += blockDim.x) {
      const int tt = o / 6, c = o % 6;
      double s = 0.0;
      for (int i = 0; i < n_qi; ++i) s += red[(i * t_tile + tt) * 6 + c];
      work[(((size_t)blockIdx.x * n_t + t0 + tt) * n_prim + k0 + a) * 6 + c] = s;
    }
  }
}

struct AccumulateStore {  // work[chunk][t][k][6]: acc += the sum
  double* acc;
  __device__ void operator()(int64_t o, double s) const { acc[o] += s; }
};

// ---------------------------------------------------------------------------------------------------------------
// Joint densities of states.  For a target q and an item (cell, tetrahedron, l1, l2) the corners are q1_i of the
// tetrahedron and q2_i = q - q1_i (integer mesh arithmetic); nu1_i = freqs[q1_i][l1], nu2_i = freqs[q2_i][l2].  The item
// gives two interpolants with corner factors c_i:
//   class 1: f_i = nu2_i - nu1_i  (the term delta(w + nu1 - nu2)),  c_i = m_i (slot 0) or m_i (n1_i - n2_i) (slot 1 + t)
//   class 2: f_i = nu1_i + nu2_i,                                   c_i = m_i           or m_i (n1_i + n2_i + 1)
// m_i = [nu1_i >= cutoff and nu2_i >= cutoff], n = 1 / expm1(h nu / k T) (0 at T = 0).  The other class-1 term,
// delta(w - nu1 + nu2), is the same sum mapped by q1 -> q - q1, l1 <-> l2 (the 6-tetrahedron set is inversion
// symmetric): the reduction doubles class 1, which also gives N2(1)'s difference.  The contribution at w is
// sum_i wt_i(w) c_i with tetra_weights' corner weights, each tetrahedron weighted 1 / (6 N).
//
// Block (x, y): JDOS_THREADS threads as blockDim.y target slots of blockDim.x (a multiple of 32) frequency points.
// Grid x: contiguous ranges of item tiles (chunks); y: groups of blockDim.y targets x tiles of blockDim.x points;
// z: the slot (0: D2, 1 + t: N2 at temperatures[t]).  Each warp of a target slot stages one sorted tile of
// blockDim.x items of its own target in shared memory (values and corner factors of both classes), then every
// thread of that slot evaluates the tile at its own frequency point (shared-memory broadcasts).  The block writes
// work[chunk][target][slot][class][f], each element by exactly one thread; chunk_reduce_kernel adds the chunks in a
// fixed order.  No atomics, and no per-item value leaves the SM.
constexpr int JDOS_THREADS = 256;

__device__ __forceinline__ double bose(double nu, double temp) {
  return temp > 0.0 ? 1.0 / expm1(TD_H_OVER_K * nu / temp) : 0.0;
}

__global__ void __launch_bounds__(JDOS_THREADS)
joint_dos_kernel(const double* __restrict__ freqs, int n_band, int n1, int n2, int n3,
                 const int32_t* __restrict__ tet, const int32_t* __restrict__ targets, int n_target,
                 const double* __restrict__ omega, int n_freq, const double* __restrict__ temps, double cutoff,
                 int64_t n_items, double* __restrict__ work) {
  // [slot y * blockDim.x + item][class][e0..e3, c0..c3]
  __shared__ double st[JDOS_THREADS][2][8];
  const int tile = blockDim.x;
  const int ti = blockIdx.y / ((n_freq + tile - 1) / tile) * blockDim.y + threadIdx.y;  // target of this slot
  const int f = blockIdx.y % ((n_freq + tile - 1) / tile) * tile + threadIdx.x;
  const bool has_target = ti < n_target;
  const bool active = has_target && f < n_freq;
  const double w = active ? omega[(size_t)ti * n_freq + f] : 0.0;
  const int slot = blockIdx.z;
  const double temp = slot > 0 ? temps[slot - 1] : 0.0;
  int qa = 0, qb = 0, qc = 0;
  if (has_target) {
    const int q = targets[ti];
    qa = q / (n2 * n3), qb = (q / n3) % n2, qc = q % n3;
  }
  double (*my)[2][8] = st + threadIdx.y * tile;
  double acc1 = 0.0, acc2 = 0.0;
  const int64_t n_tiles = (n_items + tile - 1) / tile;
  const int64_t t_end = n_tiles * (blockIdx.x + 1) / gridDim.x;
  for (int64_t t = n_tiles * blockIdx.x / gridDim.x; t < t_end; ++t) {
    const int64_t p = t * tile + threadIdx.x;
    __syncthreads();  // the previous tile has been read
    if (has_target && p < n_items) {
      const int l2 = (int)(p % n_band);
      const int64_t r = p / n_band;
      const int l1 = (int)(r % n_band);
      double e1[4], c1[4], e2[4], c2[4];
      bool any = false;
      tetrahedron_corners(tet, r / n_band, n1, n2, n3, [&](int v, int a, int b, int c) {
        int a2 = qa - a, b2 = qb - b, c2i = qc - c;
        a2 += a2 < 0 ? n1 : 0;
        b2 += b2 < 0 ? n2 : 0;
        c2i += c2i < 0 ? n3 : 0;
        const double nu1 = __ldg(freqs + (int64_t)((a * n2 + b) * n3 + c) * n_band + l1);
        const double nu2 = __ldg(freqs + (int64_t)((a2 * n2 + b2) * n3 + c2i) * n_band + l2);
        e1[v] = nu2 - nu1;
        e2[v] = nu1 + nu2;
        const bool keep = nu1 >= cutoff && nu2 >= cutoff;
        any |= keep;
        if (!keep) {
          c1[v] = c2[v] = 0.0;
        } else if (slot == 0) {
          c1[v] = c2[v] = 1.0;
        } else {
          const double b1 = bose(nu1, temp), b2v = bose(nu2, temp);
          c1[v] = b1 - b2v;
          c2[v] = b1 + b2v + 1.0;
        }
      });
      sort4(e1, c1);
      sort4(e2, c2);
      if (!any) e1[0] = e2[0] = CUDART_INF;  // every corner masked: no frequency point is evaluated
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        my[threadIdx.x][0][v] = e1[v], my[threadIdx.x][0][4 + v] = c1[v];
        my[threadIdx.x][1][v] = e2[v], my[threadIdx.x][1][4 + v] = c2[v];
      }
    }
    __syncthreads();
    if (!active) continue;
    const int n_here = (int)min((int64_t)tile, n_items - t * tile);
    for (int i = 0; i < n_here; ++i) {
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const double* s = my[i][k];
        if (!(w >= s[0] && w < s[3])) continue;
        const double e[4] = {s[0], s[1], s[2], s[3]};
        double n, g, wt[4];
        tetra_weights(w, e, n, g, wt);
        const double x = fma(wt[0], s[4], fma(wt[1], s[5], fma(wt[2], s[6], wt[3] * s[7])));
        if (k == 0) {
          acc1 += x;
        } else {
          acc2 += x;
        }
      }
    }
  }
  if (!active) return;
  const int n_slots = gridDim.z;
  double* out = work + (((size_t)blockIdx.x * n_target + ti) * n_slots + slot) * 2 * n_freq + f;
  out[0] = acc1;
  out[n_freq] = acc2;
}

struct JointDosStore {  // work[chunk][target][slot][class][f]: scale * the sum, x 2 for class 1 (both its terms)
  double* out;
  int n_freq;
  double scale;
  __device__ void operator()(int64_t o, double s) const { out[o] = s * ((o / n_freq) % 2 == 0 ? 2.0 * scale : scale); }
};

// ---------------------------------------------------------------------------------------------------------------
// Coherent one-phonon structure factors.  For row r (a scattering vector Q = q + G) and mode m,
//   F_t = sum_k coef_k exp(-W_k,t) (K . e_km) exp(-2 pi i G . x_k),  W_k,t = K^T U_k,t K / 2,
//   S+ = C (n + 1) / nu |F_t|^2,  S- = C n / nu |F_t|^2,  n = 1 / expm1(h nu / k T) (0 at T = 0),
// and S+- = 0 for nu < cutoff; C = h / (8 pi^2 amu THz) in A^2 (phonons.DISPLACEMENT_A2_AMU_THZ), applied here.
// One thread per (row, mode), grid y over tiles of SQW_T_TILE temperatures.  The thread walks the atoms once per tile:
// it reads e_km (three complex128 values), forms K . e and the phase in registers and keeps one complex F per
// temperature of its tile.  Without U (no Debye-Waller factor) F does not depend on T and one tile covers every
// temperature.  No per-(row, atom) tensor reaches global memory.
constexpr int SQW_THREADS = 256;
constexpr int SQW_T_TILE = 8;
// h / (8 pi^2 amu 1 THz) / A^2: chgnet_b200.phonons.DISPLACEMENT_A2_AMU_THZ, the same expression in the same order
constexpr double SQW_C = 6.62607015e-34 / (8 * (3.141592653589793 * 3.141592653589793) * 1.66053906660e-27 * 1e12) /
                         (1e-10 * 1e-10);

__global__ void __launch_bounds__(SQW_THREADS)
structure_factors_kernel(const double* __restrict__ freqs, const double2* __restrict__ eigvecs,
                         const double* __restrict__ kcart, const double* __restrict__ gvec,
                         const double* __restrict__ frac, const double* __restrict__ coef, const double* __restrict__ u,
                         const double* __restrict__ temps, int n_t, int n_q, int n_prim, double cutoff,
                         double* __restrict__ out) {
  const int n3 = 3 * n_prim;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_q * n3) return;
  const int row = (int)(i / n3);
  const int t0 = u ? blockIdx.y * SQW_T_TILE : 0;
  const int t_here = u ? min(SQW_T_TILE, n_t - t0) : n_t;
  const double nu = __ldg(freqs + i);
  double2* o = reinterpret_cast<double2*>(out) + (size_t)t0 * n_q * n3 + i;
  if (!(nu >= cutoff)) {
    for (int t = 0; t < t_here; ++t) o[(size_t)t * n_q * n3] = make_double2(0.0, 0.0);
    return;
  }
  const double kx = __ldg(kcart + row * 3), ky = __ldg(kcart + row * 3 + 1), kz = __ldg(kcart + row * 3 + 2);
  const double g0 = __ldg(gvec + row * 3), g1 = __ldg(gvec + row * 3 + 1), g2 = __ldg(gvec + row * 3 + 2);
  // K K^T in Voigt order with the off-diagonal terms doubled: W = acc . u / 2
  const double kk[6] = {kx * kx, ky * ky, kz * kz, 2.0 * ky * kz, 2.0 * kx * kz, 2.0 * kx * ky};
  double fr[SQW_T_TILE], fi[SQW_T_TILE];
#pragma unroll
  for (int t = 0; t < SQW_T_TILE; ++t) fr[t] = fi[t] = 0.0;
  const double2* e = eigvecs + i * n3;
  for (int k = 0; k < n_prim; ++k) {
    const double2 ex = __ldg(e + 3 * k), ey = __ldg(e + 3 * k + 1), ez = __ldg(e + 3 * k + 2);
    const double dr = fma(kx, ex.x, fma(ky, ey.x, kz * ez.x)), di = fma(kx, ex.y, fma(ky, ey.y, kz * ez.y));
    double sn, cs;  // exp(-2 pi i G . x_k) = cs - i sn
    sincospi(2.0 * fma(g0, __ldg(frac + 3 * k), fma(g1, __ldg(frac + 3 * k + 1), g2 * __ldg(frac + 3 * k + 2))), &sn,
             &cs);
    const double c = __ldg(coef + k);
    const double tr = c * fma(dr, cs, di * sn), ti = c * fma(di, cs, -dr * sn);
    if (!u) {
      fr[0] += tr;
      fi[0] += ti;
      continue;
    }
#pragma unroll
    for (int t = 0; t < SQW_T_TILE; ++t) {
      if (t >= t_here) break;
      const double* uk = u + ((size_t)(t0 + t) * n_prim + k) * 6;
      double w = 0.0;
#pragma unroll
      for (int c6 = 0; c6 < 6; ++c6) w = fma(kk[c6], __ldg(uk + c6), w);
      const double dw = exp(-0.5 * w);
      fr[t] = fma(dw, tr, fr[t]);
      fi[t] = fma(dw, ti, fi[t]);
    }
  }
  for (int t = 0; t < t_here; ++t) {
    const int tf = u ? t : 0;
    double f2 = 0.0;
#pragma unroll
    for (int j = 0; j < SQW_T_TILE; ++j)  // registers, not local memory: the index is a compile-time constant
      if (j == tf) f2 = fma(fr[j], fr[j], fi[j] * fi[j]);
    const double temp = __ldg(temps + t0 + t);
    const double n = bose(nu, temp);
    const double s = SQW_C * f2 / nu;
    o[(size_t)t * n_q * n3] = make_double2(s * (n + 1.0), s * n);
  }
}

// Broadening.  For the rows [row0, row0 + n_q) of a map whose rows form groups of group_size (row r in group
// r / group_size), out[t][g][f] += (1 / group_size) sum over the group's rows in this call and their modes of
//   S+ g(omega_f - nu) + S- g(omega_f + nu),  g(x) = exp(-x^2 / 2 sigma^2) / (sigma sqrt(2 pi)),  |x| <= 8 sigma.
// One thread per frequency point; block x = chunk + n_chunks (g - g_first + n_groups_here t), one chunk of the items
// of group g at temperature t, and block y a frequency tile.  Each tile of (row, mode) items is staged in shared memory as (nu, S+, S-) and read by every
// thread (broadcasts).  The block's sums go to work[chunk][t][g - g_first][f], each element written by exactly one
// thread: no atomics, and chunk_reduce_kernel adds the chunks in a fixed order.  No [row, mode, f] tensor exists.
constexpr int SQW_BROAD_THREADS = 256;

__global__ void __launch_bounds__(SQW_BROAD_THREADS)
broadened_spectrum_kernel(const double* __restrict__ freqs, const double2* __restrict__ weights, int n_q, int n3,
                          int n_t, int64_t row0, int group_size, int n_groups_here, const double* __restrict__ omega,
                          int n_freq, double sigma, int n_chunks, double* __restrict__ work) {
  __shared__ double st[SQW_BROAD_THREADS][3];
  const int chunk = (int)(blockIdx.x % n_chunks);
  const int gt = (int)(blockIdx.x / n_chunks);
  const int gl = gt % n_groups_here, t = gt / n_groups_here;
  const int f = blockIdx.y * blockDim.x + threadIdx.x;
  const bool active = f < n_freq;
  const double w = active ? omega[f] : 0.0;
  // the rows of group g_first + gl inside this call, relative to row0
  const int64_t g = row0 / group_size + gl;
  const int r_begin = (int)(max(g * group_size, row0) - row0);
  const int r_end = (int)(min((g + 1) * group_size, row0 + n_q) - row0);
  const int64_t n_items = (int64_t)(r_end - r_begin) * n3;
  const double2* wt = weights + (size_t)t * n_q * n3 + (size_t)r_begin * n3;
  const double* nu_g = freqs + (size_t)r_begin * n3;
  const double inv2s2 = 0.5 / (sigma * sigma), reach = 8.0 * sigma;
  const double norm = 1.0 / (sigma * 2.5066282746310002);  // sqrt(2 pi)
  double acc = 0.0;
  const int64_t tile = blockDim.x;
  const int64_t n_tiles = (n_items + tile - 1) / tile;
  const int64_t t_end = n_tiles * (chunk + 1) / n_chunks;
  for (int64_t tt = n_tiles * chunk / n_chunks; tt < t_end; ++tt) {
    const int64_t p = tt * tile + threadIdx.x;
    __syncthreads();  // the previous tile has been read
    if (p < n_items) {
      const double2 s = __ldg(wt + p);
      st[threadIdx.x][0] = __ldg(nu_g + p), st[threadIdx.x][1] = s.x, st[threadIdx.x][2] = s.y;
    }
    __syncthreads();
    if (!active) continue;
    const int n_here = (int)min(tile, n_items - tt * tile);
    for (int j = 0; j < n_here; ++j) {
      const double nu = st[j][0];
      const double xp = w - nu, xm = w + nu;
      if (fabs(xp) <= reach) acc = fma(st[j][1], exp(-xp * xp * inv2s2), acc);
      if (fabs(xm) <= reach) acc = fma(st[j][2], exp(-xm * xm * inv2s2), acc);
    }
  }
  if (!active) return;
  work[(((size_t)chunk * n_t + t) * n_groups_here + gl) * n_freq + f] = acc * norm;
}

struct SpectrumStore {  // work[chunk][t][g - g_first][f]: out[t][g][f] += scale * the sum
  double* out;
  int n_freq, n_groups_here;
  int64_t g_first, n_groups;
  double scale;
  __device__ void operator()(int64_t o, double s) const {
    const int64_t f = o % n_freq, r = o / n_freq;
    const int64_t gl = r % n_groups_here, t = r / n_groups_here;
    out[(t * n_groups + g_first + gl) * n_freq + f] += s * scale;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// The chunk reduction of the three kernels above: store(o, sum over chunks c, in chunk order, of work[c * n_out + o])
template <class Store>
__global__ void chunk_reduce_kernel(const double* __restrict__ work, int n_chunks, int64_t n_out, Store store) {
  const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n_out) return;
  double s = 0.0;
  for (int c = 0; c < n_chunks; ++c) s += work[(size_t)c * n_out + o];
  store(o, s);
}

// Checks the launch of the kernel that filled work, then launches chunk_reduce_kernel after it on the same stream
template <class Store>
cudaError_t reduce_chunks(const double* work, int n_chunks, int64_t n_out, Store store, cudaStream_t stream) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  count_launch();
  chunk_reduce_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, stream>>>(work, n_chunks, n_out, store);
  return cudaSuccess;
}

// ---------------------------------------------------------------------------------------------------------------
// Three-phonon interaction strengths.  For a target q (mesh index) and a q1 of the mesh, q2 = q - q1 on the mesh and
// G = q - q1 - q2 (integer, each component 0 or -1):
//   R[k a][k' b][k'' c] = e^{-2 pi i G.x_k} / sqrt(m_k m_k' m_k'') sum_{j' in k', j'' in k''} Phi3[k][j'][j''][a][b][c]
//                         rho_kj'(q1) rho_kj''(q2),   rho_kj(q) = (1/m_kj) sum_images e^{2 pi i q.v}
//   P[l][l1][l2] = C^3 / (36 N nu nu1 nu2) |sum e*_l(q) e_l1(q1) e_l2(q2) R|^2,   C = h / (8 pi^2 amu THz) (SQW_C),
// P = 0 when any of the three frequencies is below the cutoff.  Five stages per call, every one over all the q1 of the
// call: rho_kernel (the image averages, with the phase and the masses folded in), fc3_fourier_kernel (R, each thread one
// entry for PH3_Q1_TILE q1, so each Phi3 load serves them all), then three complex GEMMs (contract_kernel) that contract
// the modes of q, q1 and q2 in turn; the last one writes P.  Scratch: rho, and two [n_q1][3n]^3 complex buffers that R,
// the first and the second contraction take in turn.  No atomics; everything is fp64.
constexpr int PH3_THREADS = 128;
constexpr int PH3_Q1_TILE = 4;
constexpr int PH3_TILE = 32;   // GEMM output tile (both dimensions)
constexpr int PH3_KTILE = 16;  // GEMM reduction tile

struct MeshTriplet {  // q1 and q2 = target - q1 of the mesh, and G = target - q1 - q2
  int q1, q2;
  double g0, g1, g2;
  double r1[3], r2[3];  // reduced q1, q2
};

__device__ __forceinline__ MeshTriplet mesh_triplet(int target, int q1, int n1, int n2, int n3) {
  const int ta = target / (n2 * n3), tb = (target / n3) % n2, tc = target % n3;
  const int a = q1 / (n2 * n3), b = (q1 / n3) % n2, c = q1 % n3;
  int a2 = ta - a, b2 = tb - b, c2 = tc - c;
  MeshTriplet m;
  m.g0 = a2 < 0 ? -1.0 : 0.0, m.g1 = b2 < 0 ? -1.0 : 0.0, m.g2 = c2 < 0 ? -1.0 : 0.0;
  a2 += a2 < 0 ? n1 : 0;
  b2 += b2 < 0 ? n2 : 0;
  c2 += c2 < 0 ? n3 : 0;
  m.q1 = q1, m.q2 = (a2 * n2 + b2) * n3 + c2;
  m.r1[0] = (double)a / n1, m.r1[1] = (double)b / n2, m.r1[2] = (double)c / n3;
  m.r2[0] = (double)a2 / n1, m.r2[1] = (double)b2 / n2, m.r2[2] = (double)c2 / n3;
  return m;
}

// rho[q1][side][k][j], side 0: e^{-2 pi i G.x_k} rho_kj(q1) / sqrt(m_k m_s2p[j]), side 1: rho_kj(q2) / sqrt(m_s2p[j])
__global__ void __launch_bounds__(PH3_THREADS)
rho_kernel(const int32_t* __restrict__ img_ptr, const double* __restrict__ img_vec, const int32_t* __restrict__ s2p,
           const double* __restrict__ inv_sqrt_m, const double* __restrict__ frac, int n_prim, int n_super, int n1,
           int n2, int n3, int target, const int32_t* __restrict__ q1_idx, int n_q1, double2* __restrict__ rho) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t per_side = (int64_t)n_prim * n_super;
  if (i >= (int64_t)n_q1 * 2 * per_side) return;
  const int q1l = (int)(i / (2 * per_side)), side = (int)((i / per_side) % 2);
  const int k = (int)((i % per_side) / n_super), j = (int)(i % n_super);
  const MeshTriplet m = mesh_triplet(target, __ldg(q1_idx + q1l), n1, n2, n3);
  const double q0 = side == 0 ? m.r1[0] : m.r2[0], q1 = side == 0 ? m.r1[1] : m.r2[1];
  const double q2 = side == 0 ? m.r1[2] : m.r2[2];
  const size_t pair = (size_t)k * n_super + j;
  const int b = __ldg(img_ptr + pair), e = __ldg(img_ptr + pair + 1);
  double c = 0.0, s = 0.0;
  for (int t = b; t < e; ++t) {
    const double* v = img_vec + (size_t)t * 3;
    double sn, cs;
    sincospi(2.0 * fma(q0, __ldg(v), fma(q1, __ldg(v + 1), q2 * __ldg(v + 2))), &sn, &cs);
    c += cs;
    s += sn;
  }
  double w = __ldg(inv_sqrt_m + __ldg(s2p + j)) / (double)(e > b ? e - b : 1);
  if (side == 0) {
    w *= __ldg(inv_sqrt_m + k);
    double sn, cs;  // e^{-2 pi i G.x_k} = cs - i sn
    sincospi(2.0 * fma(m.g0, __ldg(frac + 3 * k), fma(m.g1, __ldg(frac + 3 * k + 1), m.g2 * __ldg(frac + 3 * k + 2))),
             &sn, &cs);
    const double cr = fma(c, cs, s * sn), ci = fma(s, cs, -c * sn);
    c = cr, s = ci;
  }
  rho[i] = make_double2(w * c, w * s);
}

// r[q1][k a][k' b][k'' c] (see above); thread: one (k, k', k'', a b c) for the PH3_Q1_TILE q1 of grid y.  Supercell
// atom j of primitive atom k' is k' n_cells + l (atom-major, as make_supercell orders it).
__global__ void __launch_bounds__(PH3_THREADS)
fc3_fourier_kernel(const double* __restrict__ fc3, const double2* __restrict__ rho, int n_prim, int n_super, int n_q1,
                   double2* __restrict__ r) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_prim * n_prim * n_prim * 27) return;
  const int abc = (int)(i % 27);
  const int64_t kkk = i / 27;
  const int kpp = (int)(kkk % n_prim), kp = (int)((kkk / n_prim) % n_prim), k = (int)(kkk / ((int64_t)n_prim * n_prim));
  const int n_cells = n_super / n_prim;
  const int q0 = blockIdx.y * PH3_Q1_TILE;
  const int nq = min(PH3_Q1_TILE, n_q1 - q0);
  double ar[PH3_Q1_TILE], ai[PH3_Q1_TILE];
#pragma unroll
  for (int t = 0; t < PH3_Q1_TILE; ++t) ar[t] = ai[t] = 0.0;
  const size_t side = (size_t)n_prim * n_super;
  const double2* rho_k = rho + (size_t)q0 * 2 * side + (size_t)k * n_super;
  for (int lp = 0; lp < n_cells; ++lp) {
    const int jp = kp * n_cells + lp;
    const double* f = fc3 + (((size_t)k * n_super + jp) * n_super + (size_t)kpp * n_cells) * 27 + abc;
    double br[PH3_Q1_TILE], bi[PH3_Q1_TILE];
#pragma unroll
    for (int t = 0; t < PH3_Q1_TILE; ++t) br[t] = bi[t] = 0.0;
    for (int lpp = 0; lpp < n_cells; ++lpp) {
      const double x = __ldg(f + (size_t)lpp * 27);
#pragma unroll
      for (int t = 0; t < PH3_Q1_TILE; ++t) {
        if (t >= nq) break;
        const double2 p2 = __ldg(rho_k + (size_t)t * 2 * side + side + kpp * n_cells + lpp);
        br[t] = fma(x, p2.x, br[t]);
        bi[t] = fma(x, p2.y, bi[t]);
      }
    }
#pragma unroll
    for (int t = 0; t < PH3_Q1_TILE; ++t) {
      if (t >= nq) break;
      const double2 p1 = __ldg(rho_k + (size_t)t * 2 * side + jp);
      ar[t] = fma(p1.x, br[t], fma(-p1.y, bi[t], ar[t]));
      ai[t] = fma(p1.x, bi[t], fma(p1.y, br[t], ai[t]));
    }
  }
  const int n3 = 3 * n_prim;
  const int a = abc / 9, b = (abc / 3) % 3, c = abc % 3;
  const size_t o = ((size_t)(3 * k + a) * n3 + 3 * kp + b) * n3 + 3 * kpp + c;
  const size_t n33 = (size_t)n3 * n3 * n3;
#pragma unroll
  for (int t = 0; t < PH3_Q1_TILE; ++t) {
    if (t >= nq) break;
    r[(size_t)(q0 + t) * n33 + o] = make_double2(ar[t], ai[t]);
  }
}

// The three contractions as complex GEMMs C[m][n] = sum_k A(m, k) B(k, n), one q1 per grid z and PH3_TILE^2 outputs per
// block, e the mode-major eigenvectors (e[q][mode][k a]):
//   STAGE 0: A = conj(e[target]) [l][k a], B = R [k a][k' b, k'' c]          -> c1 [l][k' b, k'' c]
//   STAGE 1: per l (sub), A = e[q1] [l1][k' b], B = c1[l] [k' b][k'' c]       -> c2 [l][l1][k'' c]
//   STAGE 2: A = c2 [l l1][k'' c], B(k, n) = e[q2][n][k], and P = C^3 / (36 N nu nu1 nu2) |C|^2 (0 below the cutoff)
template <int STAGE>
__global__ void __launch_bounds__(256)
contract_kernel(const double2* __restrict__ eig, const double* __restrict__ freqs, int n_prim, int n1, int n2, int n3m,
                int target, const int32_t* __restrict__ q1_idx, double cutoff, double p_scale,
                const double2* __restrict__ in, double2* __restrict__ out, double* __restrict__ p) {
  __shared__ double2 sa[PH3_KTILE][PH3_TILE];
  __shared__ double2 sb[PH3_KTILE][PH3_TILE + 1];
  const int n3 = 3 * n_prim;
  const size_t n33 = (size_t)n3 * n3 * n3;
  const int q1l = blockIdx.z;
  const MeshTriplet mt = mesh_triplet(target, __ldg(q1_idx + q1l), n1, n2, n3m);
  const int big = STAGE == 0 ? n3 * n3 : n3;  // N of stage 0, M of stage 2
  const int rows = STAGE == 2 ? n3 * n3 : n3, cols = STAGE == 0 ? big : n3;
  const int tm = (rows + PH3_TILE - 1) / PH3_TILE, tn = (cols + PH3_TILE - 1) / PH3_TILE;
  const int sub = blockIdx.x / (tm * tn);
  const int m0 = (blockIdx.x % (tm * tn)) / tn * PH3_TILE, c0 = blockIdx.x % tn * PH3_TILE;
  const double2* a_base;
  const double2* b_base;
  if constexpr (STAGE == 0) {
    a_base = eig + (size_t)target * n3 * n3;
    b_base = in + (size_t)q1l * n33;
  } else if constexpr (STAGE == 1) {
    a_base = eig + (size_t)mt.q1 * n3 * n3;
    b_base = in + (size_t)q1l * n33 + (size_t)sub * n3 * n3;
  } else {
    a_base = in + (size_t)q1l * n33;
    b_base = eig + (size_t)mt.q2 * n3 * n3;
  }
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  double cr[2][2] = {{0.0, 0.0}, {0.0, 0.0}}, ci[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
  for (int k0 = 0; k0 < n3; k0 += PH3_KTILE) {
    __syncthreads();  // the previous tiles have been read
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int e = threadIdx.x + 256 * r;
      const int am = e / PH3_KTILE, ak = e % PH3_KTILE;  // A(m0 + am, k0 + ak), k fastest
      double2 x = make_double2(0.0, 0.0);
      if (m0 + am < rows && k0 + ak < n3) {
        x = __ldg(a_base + (size_t)(m0 + am) * n3 + k0 + ak);
        if constexpr (STAGE == 0) x.y = -x.y;
      }
      sa[ak][am] = x;
      double2 y = make_double2(0.0, 0.0);
      if constexpr (STAGE == 2) {  // B(k, n) = e[q2][n][k]: k fastest
        const int bn = e / PH3_KTILE, bk = e % PH3_KTILE;
        if (c0 + bn < cols && k0 + bk < n3) y = __ldg(b_base + (size_t)(c0 + bn) * n3 + k0 + bk);
        sb[bk][bn] = y;
      } else {
        const int bk = e / PH3_TILE, bn = e % PH3_TILE;
        if (c0 + bn < cols && k0 + bk < n3) y = __ldg(b_base + (size_t)(k0 + bk) * cols + c0 + bn);
        sb[bk][bn] = y;
      }
    }
    __syncthreads();
    const int kn = min(PH3_KTILE, n3 - k0);
    for (int kk = 0; kk < kn; ++kk) {
      const double2 a0 = sa[kk][ty], a1 = sa[kk][ty + 16];
      const double2 b0 = sb[kk][tx], b1 = sb[kk][tx + 16];
      cr[0][0] = fma(a0.x, b0.x, fma(-a0.y, b0.y, cr[0][0]));
      ci[0][0] = fma(a0.x, b0.y, fma(a0.y, b0.x, ci[0][0]));
      cr[0][1] = fma(a0.x, b1.x, fma(-a0.y, b1.y, cr[0][1]));
      ci[0][1] = fma(a0.x, b1.y, fma(a0.y, b1.x, ci[0][1]));
      cr[1][0] = fma(a1.x, b0.x, fma(-a1.y, b0.y, cr[1][0]));
      ci[1][0] = fma(a1.x, b0.y, fma(a1.y, b0.x, ci[1][0]));
      cr[1][1] = fma(a1.x, b1.x, fma(-a1.y, b1.y, cr[1][1]));
      ci[1][1] = fma(a1.x, b1.y, fma(a1.y, b1.x, ci[1][1]));
    }
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int m = m0 + ty + 16 * i, c = c0 + tx + 16 * j;
      if (m >= rows || c >= cols) continue;
      if constexpr (STAGE == 0) {
        out[(size_t)q1l * n33 + (size_t)m * cols + c] = make_double2(cr[i][j], ci[i][j]);
      } else if constexpr (STAGE == 1) {
        out[(size_t)q1l * n33 + ((size_t)sub * n3 + m) * n3 + c] = make_double2(cr[i][j], ci[i][j]);
      } else {
        const double nu = __ldg(freqs + (size_t)target * n3 + m / n3);
        const double nu1 = __ldg(freqs + (size_t)mt.q1 * n3 + m % n3);
        const double nu2 = __ldg(freqs + (size_t)mt.q2 * n3 + c);
        const bool keep = nu >= cutoff && nu1 >= cutoff && nu2 >= cutoff;
        p[(size_t)q1l * n33 + (size_t)m * n3 + c] =
            keep ? p_scale * fma(cr[i][j], cr[i][j], ci[i][j] * ci[i][j]) / (nu * nu1 * nu2) : 0.0;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Imaginary self-energy.  For the target q and an item (q1, l1, l2) of the call, vertex q1 enters the tetrahedron
// averages of the three deltas with the weights
//   g(w) = 1/6 sum over the 24 (tetrahedron, corner) with that corner at q1 of tetra_weights' corner weight,
// for the corner values f = nu1 + nu2 (g2: d(w - nu1 - nu2)), nu2 - nu1 (g1+: d(w + nu1 - nu2)) and nu1 - nu2 (g1-:
// d(w - nu1 + nu2)), nu1 = freqs[q1'][l1], nu2 = freqs[q - q1'][l2] at each corner q1'.  (1/N) sum_q1 g reproduces the
// tetrahedron sums of chg_joint_dos.  An item with nu1 or nu2 below the cutoff has weight 0.
// ise_weights_kernel: one thread per item; it sorts the three corner sets of each of the 24 tetrahedra once and
// evaluates them at every band frequency w_l (>= cutoff) inside their range, writing (g2, g1+ - g1-) to
// wts[q1][l][l1][l2] (the layout of P), each element by its own thread.  ise_accumulate_kernel: block (chunk, l, tile
// of ISE_T_TILE temperatures) adds 18 pi / h^2 P [(1 + n1 + n2) g2 + (n1 - n2) (g1+ - g1-)] over its chunk of items in
// a fixed order and writes work[chunk][t][l]; chunk_reduce_kernel adds the chunks in chunk order to gamma.  The
// weights depend on the frequencies only and are formed once per call for every temperature.  No atomics.
constexpr int ISE_THREADS = 256;
constexpr int ISE_T_TILE = 8;
// 18 pi / h^2 with h in eV/THz: chgnet_b200.phonons.H_EV_PER_THZ, the same expression in the same order
constexpr double ISE_H = 6.62607015e-34 / 1.602176634e-19 * 1e12;

// wt[p] for a run-time index p, from registers
__device__ __forceinline__ double corner_weight(const double (&wt)[4], int p) {
  return p == 0 ? wt[0] : (p == 1 ? wt[1] : (p == 2 ? wt[2] : wt[3]));
}

// SPLIT false: wts [q1][l][l1][l2] of (g2, g1+ - g1-) (chg_imag_self_energy).  SPLIT true: wts holds three planes
// of doubles [3][n_q1][l][l1][l2], g2, g1+ and g1- (chg_collision_rows).
template <bool SPLIT>
__global__ void __launch_bounds__(ISE_THREADS)
ise_weights_kernel(const double* __restrict__ freqs, int n_band, int n1, int n2, int n3,
                   const int32_t* __restrict__ tet, int target, const double* __restrict__ omega,
                   const int32_t* __restrict__ q1_idx, int n_q1, double cutoff, double2* __restrict__ wts) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t nb2 = (int64_t)n_band * n_band;
  if (i >= (int64_t)n_q1 * nb2) return;
  const int q1l = (int)(i / nb2), l1 = (int)((i / n_band) % n_band), l2 = (int)(i % n_band);
  double2* w_out = wts + (size_t)q1l * n_band * nb2 + (size_t)(i % nb2);
  double* w_plane = reinterpret_cast<double*>(wts) + (size_t)q1l * n_band * nb2 + (size_t)(i % nb2);
  const size_t plane = (size_t)n_q1 * n_band * nb2;
  if constexpr (SPLIT) {
    for (int l = 0; l < n_band; ++l) {
      w_plane[(size_t)l * nb2] = 0.0;
      w_plane[plane + (size_t)l * nb2] = 0.0;
      w_plane[2 * plane + (size_t)l * nb2] = 0.0;
    }
  } else {
    for (int l = 0; l < n_band; ++l) w_out[(size_t)l * nb2] = make_double2(0.0, 0.0);
  }
  const int q1 = __ldg(q1_idx + q1l);
  const int ta = target / (n2 * n3), tb = (target / n3) % n2, tc = target % n3;
  const auto nu_pair = [&](int a, int b, int c, double& nu1, double& nu2) {
    int a2 = ta - a, b2 = tb - b, c2 = tc - c;
    a2 += a2 < 0 ? n1 : 0;
    b2 += b2 < 0 ? n2 : 0;
    c2 += c2 < 0 ? n3 : 0;
    nu1 = __ldg(freqs + (int64_t)((a * n2 + b) * n3 + c) * n_band + l1);
    nu2 = __ldg(freqs + (int64_t)((a2 * n2 + b2) * n3 + c2) * n_band + l2);
  };
  const int qa = q1 / (n2 * n3), qb = (q1 / n3) % n2, qc = q1 % n3;
  double nu1, nu2;
  nu_pair(qa, qb, qc, nu1, nu2);
  if (!(nu1 >= cutoff && nu2 >= cutoff)) return;
  for (int tv = 0; tv < 24; ++tv) {
    const int it = tv / 4, v = tv % 4;
    const int32_t* o = tet + (it * 4 + v) * 3;
    // the cell whose corner v of tetrahedron it is q1
    int ca = qa - __ldg(o), cb = qb - __ldg(o + 1), cc = qc - __ldg(o + 2);
    ca += ca < 0 ? n1 : 0;
    cb += cb < 0 ? n2 : 0;
    cc += cc < 0 ? n3 : 0;
    double e2[4], ep[4], em[4];
    int x2[4], xp[4], xm[4];
    tetrahedron_corners(tet, ((int64_t)(ca * n2 + cb) * n3 + cc) * 6 + it, n1, n2, n3, [&](int u, int a, int b, int c) {
      double v1, v2;
      nu_pair(a, b, c, v1, v2);
      e2[u] = v1 + v2, ep[u] = v2 - v1, em[u] = v1 - v2;
      x2[u] = xp[u] = xm[u] = u;
    });
    sort4(e2, x2);
    sort4(ep, xp);
    sort4(em, xm);
    int p2 = 0, pp = 0, pm = 0;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      p2 = x2[u] == v ? u : p2;
      pp = xp[u] == v ? u : pp;
      pm = xm[u] == v ? u : pm;
    }
    for (int l = 0; l < n_band; ++l) {
      const double w = __ldg(omega + l);
      if (!(w >= cutoff)) continue;
      const bool h2 = w >= e2[0] && w < e2[3], hp = w >= ep[0] && w < ep[3], hm = w >= em[0] && w < em[3];
      if (!(h2 || hp || hm)) continue;
      double n, g, wt[4], d2 = 0.0, d1 = 0.0, dm = 0.0;
      if (h2) {
        tetra_weights(w, e2, n, g, wt);
        d2 = corner_weight(wt, p2);
      }
      if (hp) {
        tetra_weights(w, ep, n, g, wt);
        d1 = corner_weight(wt, pp);
      }
      if (hm) {
        tetra_weights(w, em, n, g, wt);
        if constexpr (SPLIT) {
          dm = corner_weight(wt, pm);
        } else {
          d1 -= corner_weight(wt, pm);
        }
      }
      if constexpr (SPLIT) {
        double* o = w_plane + (size_t)l * nb2;
        o[0] = fma(d2, 1.0 / 6.0, o[0]);
        o[plane] = fma(d1, 1.0 / 6.0, o[plane]);
        o[2 * plane] = fma(dm, 1.0 / 6.0, o[2 * plane]);
      } else {
        double2 acc = w_out[(size_t)l * nb2];
        acc.x = fma(d2, 1.0 / 6.0, acc.x);
        acc.y = fma(d1, 1.0 / 6.0, acc.y);
        w_out[(size_t)l * nb2] = acc;
      }
    }
  }
}

__global__ void __launch_bounds__(ISE_THREADS)
ise_accumulate_kernel(const double* __restrict__ freqs, int n_band, int n1, int n2, int n3, int target,
                      const double* __restrict__ omega, const int32_t* __restrict__ q1_idx, int n_q1,
                      const double* __restrict__ p, const double2* __restrict__ wts, const double* __restrict__ temps,
                      int n_t, double cutoff, double* __restrict__ work) {
  __shared__ double red[ISE_THREADS][ISE_T_TILE];
  const int l = blockIdx.y, t0 = blockIdx.z * ISE_T_TILE;
  const int t_here = min(ISE_T_TILE, n_t - t0);
  const int64_t nb2 = (int64_t)n_band * n_band, n_items = (int64_t)n_q1 * nb2;
  const int64_t begin = n_items * blockIdx.x / gridDim.x, end = n_items * (blockIdx.x + 1) / gridDim.x;
  double acc[ISE_T_TILE];
#pragma unroll
  for (int t = 0; t < ISE_T_TILE; ++t) acc[t] = 0.0;
  double tt[ISE_T_TILE];
#pragma unroll
  for (int t = 0; t < ISE_T_TILE; ++t) tt[t] = t < t_here ? __ldg(temps + t0 + t) : 0.0;
  const int ta = target / (n2 * n3), tb = (target / n3) % n2, tc = target % n3;
  if (__ldg(omega + l) >= cutoff) {
    for (int64_t i = begin + threadIdx.x; i < end; i += ISE_THREADS) {
      const int q1l = (int)(i / nb2);
      const size_t at = ((size_t)q1l * n_band + l) * nb2 + (size_t)(i % nb2);
      const double2 w = __ldg(wts + at);
      if (w.x == 0.0 && w.y == 0.0) continue;
      const double pv = __ldg(p + at);
      if (pv == 0.0) continue;
      const int l1 = (int)((i / n_band) % n_band), l2 = (int)(i % n_band);
      const int q1 = __ldg(q1_idx + q1l);
      const int a = q1 / (n2 * n3), b = (q1 / n3) % n2, c = q1 % n3;
      int a2 = ta - a, b2 = tb - b, c2 = tc - c;
      a2 += a2 < 0 ? n1 : 0;
      b2 += b2 < 0 ? n2 : 0;
      c2 += c2 < 0 ? n3 : 0;
      const double nu1 = __ldg(freqs + (int64_t)q1 * n_band + l1);
      const double nu2 = __ldg(freqs + (int64_t)((a2 * n2 + b2) * n3 + c2) * n_band + l2);
#pragma unroll
      for (int t = 0; t < ISE_T_TILE; ++t) {
        if (t >= t_here) break;
        const double b1 = bose(nu1, tt[t]), b2v = bose(nu2, tt[t]);
        acc[t] = fma(pv, fma(1.0 + b1 + b2v, w.x, (b1 - b2v) * w.y), acc[t]);
      }
    }
  }
#pragma unroll
  for (int t = 0; t < ISE_T_TILE; ++t) red[threadIdx.x][t] = acc[t];
  __syncthreads();
  if (threadIdx.x < t_here) {
    double s = 0.0;
    for (int i = 0; i < ISE_THREADS; ++i) s += red[i][threadIdx.x];
    work[((size_t)blockIdx.x * n_t + t0 + threadIdx.x) * n_band + l] = s * (18.0 * 3.141592653589793 / (ISE_H * ISE_H));
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Collision-matrix rows.  For the target q, a vertex q1 of the call, q2 = q - q1 and s(nu) = sinh(h nu / 2 k T), the
// four role sums of (l, b), each times 2 pi 18 pi / h^2:
//   A = -sum_k P[l][b][k] (g2 + g1-)[l][b][k] / s(nu2_k)    B = +sum_k P[l][b][k] g1+[l][b][k] / s(nu2_k)
//   C = -sum_k P[l][k][b] (g2 + g1+)[l][k][b] / s(nu1_k)    D = +sum_k P[l][k][b] g1-[l][k][b] / s(nu1_k)
// (nu1 at q1, nu2 at q2) go to out[role][t][l][q1][b], q1 the mesh index.  collision_rows_kernel: block (q1 of the
// call, tile of COLL_T_TILE temperatures); it stages 1 / s(nu1) and 1 / s(nu2) of the tile in shared memory (0 below
// the cutoff and at T = 0), then each thread owns whole (l, b) pairs and sums k in ascending order for all four roles
// and the tile's temperatures.  Every output element is written by one thread, no atomics.
constexpr int COLL_THREADS = 256;
constexpr int COLL_T_TILE = 4;
constexpr int COLL_MAX_BAND = 768;  // the staged 1 / s: 2 x COLL_T_TILE x n_band doubles within 48 KiB

__global__ void __launch_bounds__(COLL_THREADS)
collision_rows_kernel(const double* __restrict__ freqs, int n_band, int n1, int n2, int n3, int target,
                      const int32_t* __restrict__ q1_idx, int n_q1, const double* __restrict__ p,
                      const double* __restrict__ wts, const double* __restrict__ temps, int n_t, double cutoff,
                      double* __restrict__ out) {
  extern __shared__ double inv_s[];  // [2][COLL_T_TILE][n_band]: side 0 at q1, side 1 at q2
  const int q1l = blockIdx.x, t0 = blockIdx.y * COLL_T_TILE;
  const int t_here = min(COLL_T_TILE, n_t - t0);
  const int n_mesh = n1 * n2 * n3;
  const int q1 = __ldg(q1_idx + q1l);
  const int ta = target / (n2 * n3), tb = (target / n3) % n2, tc = target % n3;
  int a2 = ta - q1 / (n2 * n3), b2 = tb - (q1 / n3) % n2, c2 = tc - q1 % n3;
  a2 += a2 < 0 ? n1 : 0;
  b2 += b2 < 0 ? n2 : 0;
  c2 += c2 < 0 ? n3 : 0;
  const int q2 = (a2 * n2 + b2) * n3 + c2;
  for (int i = threadIdx.x; i < 2 * COLL_T_TILE * n_band; i += COLL_THREADS) {
    const int side = i / (COLL_T_TILE * n_band), t = (i / n_band) % COLL_T_TILE, k = i % n_band;
    const double nu = __ldg(freqs + (int64_t)(side == 0 ? q1 : q2) * n_band + k);
    const double temp = t < t_here ? __ldg(temps + t0 + t) : 0.0;
    inv_s[i] = nu >= cutoff && temp > 0.0 ? 1.0 / sinh(0.5 * TD_H_OVER_K * nu / temp) : 0.0;
  }
  __syncthreads();
  const int64_t nb2 = (int64_t)n_band * n_band, n_w = (int64_t)n_q1 * n_band * nb2;
  const double* pq = p + (size_t)q1l * n_band * nb2;
  const double* g2 = wts + (size_t)q1l * n_band * nb2;
  const double* gp = g2 + n_w;
  const double* gm = g2 + 2 * n_w;
  const double scale = 2.0 * 3.141592653589793 * (18.0 * 3.141592653589793 / (ISE_H * ISE_H));
  for (int64_t i = threadIdx.x; i < nb2; i += COLL_THREADS) {
    const int l = (int)(i / n_band), b = (int)(i % n_band);
    double ra[COLL_T_TILE], rb[COLL_T_TILE], rc[COLL_T_TILE], rd[COLL_T_TILE];
#pragma unroll
    for (int t = 0; t < COLL_T_TILE; ++t) ra[t] = rb[t] = rc[t] = rd[t] = 0.0;
    const size_t row = (size_t)l * nb2 + (size_t)b * n_band;  // [l][b][k]
    const size_t col = (size_t)l * nb2 + b;                    // [l][k][b] at k = 0
    for (int k = 0; k < n_band; ++k) {
      const double pr = __ldg(pq + row + k), pc = __ldg(pq + col + (size_t)k * n_band);
      // P is 0 wherever a mode is below the cutoff; the weights are 0 off the delta functions' support
      const double x2 = pr * (__ldg(g2 + row + k) + __ldg(gm + row + k)), xp = pr * __ldg(gp + row + k);
      const double y2 = pc * (__ldg(g2 + col + (size_t)k * n_band) + __ldg(gp + col + (size_t)k * n_band));
      const double ym = pc * __ldg(gm + col + (size_t)k * n_band);
#pragma unroll
      for (int t = 0; t < COLL_T_TILE; ++t) {
        const double s2 = inv_s[(COLL_T_TILE + t) * n_band + k], s1 = inv_s[t * n_band + k];
        ra[t] = fma(x2, s2, ra[t]);
        rb[t] = fma(xp, s2, rb[t]);
        rc[t] = fma(y2, s1, rc[t]);
        rd[t] = fma(ym, s1, rd[t]);
      }
    }
#pragma unroll
    for (int t = 0; t < COLL_T_TILE; ++t) {
      if (t >= t_here) break;
      const size_t o = (((size_t)(t0 + t) * n_band + l) * n_mesh + q1) * n_band + b;
      const size_t role = (size_t)n_t * n_band * n_mesh * n_band;
      out[o] = -scale * ra[t];
      out[role + o] = scale * rb[t];
      out[2 * role + o] = -scale * rc[t];
      out[3 * role + o] = scale * rd[t];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Self-energy spectrum.  gamma[t][l][f] += 18 pi / h^2 sum over the items (q1, l1, l2) of the call of
//   P[q1][l][l1][l2] [(1 + n1 + n2) g2(w_f) + (n1 - n2) (g1+ - g1-)(w_f)]
// with the vertex weights of ise_weights_kernel, evaluated at the points w_f shared by every band instead of at the
// band frequencies; a point below the cutoff gets 0.  Block (chunk of item tiles, tile of SE_F_TILE points x tile of
// SE_L_TILE bands, tile of SE_T_TILE temperatures), SE_THREADS threads, per tile of SE_ITEMS items:
//   1. thread (item, tv) sorts the three corner sets (nu1 + nu2, nu2 - nu1, nu1 - nu2) of the tetrahedron-corner tv
//      around q1 into shared memory, with the position of q1 in each; the other threads stage P[q1][l][l1][l2] of the
//      band tile and the occupation factors 1 + n1 + n2 and n1 - n2 of each item at the tile's temperatures;
//   2. thread (item = warp, point = lane) walks its item's 24 x 3 sets in the order of ise_weights_kernel and
//      writes (g2, g1+ - g1-) at its point; the warp marks an item with no weight at any point of the tile;
//   3. thread (band = warp + 8 j, point = lane) adds P times the occupation-weighted weights over the tile's items in
//      order, skipping the marked items and P = 0 (both uniform across the warp).
// The block writes work[chunk][t][l][f], each element by one thread; chunk_reduce_kernel adds the chunks in chunk order
// to gamma.  No atomics, and no per-(item, point) value leaves the SM.
constexpr int SE_THREADS = 256;
constexpr int SE_ITEMS = 8;                            // items per staged tile: one warp each in step 2
constexpr int SE_F_TILE = 32;                          // points per block: one lane each
constexpr int SE_L_PER = 4;                            // bands per thread in step 3
constexpr int SE_L_TILE = SE_L_PER * SE_THREADS / 32;  // bands per block
constexpr int SE_T_TILE = 4;                           // temperatures per block
constexpr int SE_SORTERS = SE_ITEMS * 24;              // step-1 threads that sort; the rest stage P and occupations

__global__ void __launch_bounds__(SE_THREADS)
self_energy_spectrum_kernel(const double* __restrict__ freqs, int n_band, int n1, int n2, int n3,
                            const int32_t* __restrict__ tet, int target, const double* __restrict__ omega, int n_freq,
                            const int32_t* __restrict__ q1_idx, int n_q1, const double* __restrict__ p,
                            const double* __restrict__ temps, int n_t, double cutoff, double* __restrict__ work) {
  __shared__ double s_e[SE_ITEMS][24][3][4];        // sorted corner values per (item, tv, class)
  __shared__ int8_t s_pos[SE_ITEMS][24][3];         // the position of q1 among them
  __shared__ double s_p[SE_ITEMS][SE_L_TILE];       // P[q1][l0 + j][l1][l2]
  __shared__ double s_occ[SE_ITEMS][SE_T_TILE][2];  // 1 + n1 + n2, n1 - n2
  __shared__ double2 s_w[SE_ITEMS][SE_F_TILE];      // (g2, g1+ - g1-) at the tile's points
  __shared__ int s_any[SE_ITEMS];
  const int f_tiles = (n_freq + SE_F_TILE - 1) / SE_F_TILE;
  const int f0 = (blockIdx.y % f_tiles) * SE_F_TILE, l0 = (blockIdx.y / f_tiles) * SE_L_TILE;
  const int t0 = blockIdx.z * SE_T_TILE;
  const int t_here = min(SE_T_TILE, n_t - t0);
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int f = f0 + lane;
  const double w = f < n_freq ? __ldg(omega + f) : 0.0;
  const bool live_point = f < n_freq && w >= cutoff;
  const int64_t nb2 = (int64_t)n_band * n_band, n_items = (int64_t)n_q1 * nb2;
  const int ta = target / (n2 * n3), tb = (target / n3) % n2, tc = target % n3;
  double acc[SE_L_PER][SE_T_TILE];
#pragma unroll
  for (int j = 0; j < SE_L_PER; ++j)
#pragma unroll
    for (int t = 0; t < SE_T_TILE; ++t) acc[j][t] = 0.0;
  const int64_t n_tiles = (n_items + SE_ITEMS - 1) / SE_ITEMS;
  const int64_t t_end = n_tiles * (blockIdx.x + 1) / gridDim.x;
  for (int64_t tile = n_tiles * blockIdx.x / gridDim.x; tile < t_end; ++tile) {
    __syncthreads();  // the previous tile has been read
    if (threadIdx.x < SE_SORTERS) {
      const int it = threadIdx.x / 24, tv = threadIdx.x % 24;
      const int64_t i = tile * SE_ITEMS + it;
      double e2[4], ep[4], em[4];
      int x2[4], xp[4], xm[4];
      bool live = false;
      if (i < n_items) {
        const int q1 = __ldg(q1_idx + (int)(i / nb2)), l1 = (int)((i / n_band) % n_band), l2 = (int)(i % n_band);
        const auto nu_pair = [&](int a, int b, int c, double& nu1, double& nu2) {
          int a2 = ta - a, b2 = tb - b, c2 = tc - c;
          a2 += a2 < 0 ? n1 : 0;
          b2 += b2 < 0 ? n2 : 0;
          c2 += c2 < 0 ? n3 : 0;
          nu1 = __ldg(freqs + (int64_t)((a * n2 + b) * n3 + c) * n_band + l1);
          nu2 = __ldg(freqs + (int64_t)((a2 * n2 + b2) * n3 + c2) * n_band + l2);
        };
        const int qa = q1 / (n2 * n3), qb = (q1 / n3) % n2, qc = q1 % n3;
        double nu1, nu2;
        nu_pair(qa, qb, qc, nu1, nu2);
        live = nu1 >= cutoff && nu2 >= cutoff;
        if (live) {
          const int iv = tv / 4, v = tv % 4;
          const int32_t* o = tet + (iv * 4 + v) * 3;
          // the cell whose corner v of tetrahedron iv is q1
          int ca = qa - __ldg(o), cb = qb - __ldg(o + 1), cc = qc - __ldg(o + 2);
          ca += ca < 0 ? n1 : 0;
          cb += cb < 0 ? n2 : 0;
          cc += cc < 0 ? n3 : 0;
          tetrahedron_corners(tet, ((int64_t)(ca * n2 + cb) * n3 + cc) * 6 + iv, n1, n2, n3,
                              [&](int u, int a, int b, int c) {
                                double v1, v2;
                                nu_pair(a, b, c, v1, v2);
                                e2[u] = v1 + v2, ep[u] = v2 - v1, em[u] = v1 - v2;
                                x2[u] = xp[u] = xm[u] = u;
                              });
          sort4(e2, x2);
          sort4(ep, xp);
          sort4(em, xm);
          int p2 = 0, pp = 0, pm = 0;
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            p2 = x2[u] == v ? u : p2;
            pp = xp[u] == v ? u : pp;
            pm = xm[u] == v ? u : pm;
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            s_e[it][tv][0][u] = e2[u];
            s_e[it][tv][1][u] = ep[u];
            s_e[it][tv][2][u] = em[u];
          }
          s_pos[it][tv][0] = (int8_t)p2, s_pos[it][tv][1] = (int8_t)pp, s_pos[it][tv][2] = (int8_t)pm;
        }
      }
      if (!live) {  // an empty range: no point is evaluated
#pragma unroll
        for (int k = 0; k < 3; ++k) s_e[it][tv][k][0] = CUDART_INF;
      }
    } else {
      for (int k = threadIdx.x - SE_SORTERS; k < SE_ITEMS * SE_L_TILE; k += SE_THREADS - SE_SORTERS) {
        const int it = k / SE_L_TILE, l = l0 + k % SE_L_TILE;
        const int64_t i = tile * SE_ITEMS + it;
        s_p[it][k % SE_L_TILE] =
            i < n_items && l < n_band ? __ldg(p + ((i / nb2) * n_band + l) * nb2 + (i % nb2)) : 0.0;
      }
      for (int k = threadIdx.x - SE_SORTERS; k < SE_ITEMS * SE_T_TILE; k += SE_THREADS - SE_SORTERS) {
        const int it = k / SE_T_TILE, t = k % SE_T_TILE;
        const int64_t i = tile * SE_ITEMS + it;
        double b1 = 0.0, b2v = 0.0;
        if (i < n_items && t < t_here) {
          const int q1 = __ldg(q1_idx + (int)(i / nb2)), l1 = (int)((i / n_band) % n_band), l2 = (int)(i % n_band);
          int a2 = ta - q1 / (n2 * n3), b2 = tb - (q1 / n3) % n2, c2 = tc - q1 % n3;
          a2 += a2 < 0 ? n1 : 0;
          b2 += b2 < 0 ? n2 : 0;
          c2 += c2 < 0 ? n3 : 0;
          const double temp = __ldg(temps + t0 + t);
          b1 = bose(__ldg(freqs + (int64_t)q1 * n_band + l1), temp);
          b2v = bose(__ldg(freqs + (int64_t)((a2 * n2 + b2) * n3 + c2) * n_band + l2), temp);
        }
        s_occ[it][t][0] = 1.0 + b1 + b2v;
        s_occ[it][t][1] = b1 - b2v;
      }
    }
    __syncthreads();
    {
      double gx = 0.0, gy = 0.0;
      if (live_point) {
        for (int tv = 0; tv < 24; ++tv) {
          const double* s2 = s_e[warp][tv][0];
          const double* sp = s_e[warp][tv][1];
          const double* sm = s_e[warp][tv][2];
          const bool h2 = w >= s2[0] && w < s2[3], hp = w >= sp[0] && w < sp[3], hm = w >= sm[0] && w < sm[3];
          if (!(h2 || hp || hm)) continue;
          double n, g, wt[4], d2 = 0.0, d1 = 0.0;
          if (h2) {
            const double e[4] = {s2[0], s2[1], s2[2], s2[3]};
            tetra_weights(w, e, n, g, wt);
            d2 = corner_weight(wt, s_pos[warp][tv][0]);
          }
          if (hp) {
            const double e[4] = {sp[0], sp[1], sp[2], sp[3]};
            tetra_weights(w, e, n, g, wt);
            d1 = corner_weight(wt, s_pos[warp][tv][1]);
          }
          if (hm) {
            const double e[4] = {sm[0], sm[1], sm[2], sm[3]};
            tetra_weights(w, e, n, g, wt);
            d1 -= corner_weight(wt, s_pos[warp][tv][2]);
          }
          gx = fma(d2, 1.0 / 6.0, gx);
          gy = fma(d1, 1.0 / 6.0, gy);
        }
      }
      s_w[warp][lane] = make_double2(gx, gy);
      const bool any = __any_sync(0xffffffffu, gx != 0.0 || gy != 0.0);
      if (lane == 0) s_any[warp] = any;
    }
    __syncthreads();
    for (int it = 0; it < SE_ITEMS; ++it) {
      if (!s_any[it]) continue;
      const double2 g = s_w[it][lane];
      double c2[SE_T_TILE], c1[SE_T_TILE];
#pragma unroll
      for (int t = 0; t < SE_T_TILE; ++t) c2[t] = s_occ[it][t][0], c1[t] = s_occ[it][t][1];
#pragma unroll
      for (int j = 0; j < SE_L_PER; ++j) {
        const double pv = s_p[it][warp + 8 * j];
        if (pv == 0.0) continue;
#pragma unroll
        for (int t = 0; t < SE_T_TILE; ++t) acc[j][t] = fma(pv, fma(c2[t], g.x, c1[t] * g.y), acc[j][t]);
      }
    }
  }
  if (f >= n_freq) return;
  const double scale = 18.0 * 3.141592653589793 / (ISE_H * ISE_H);
#pragma unroll
  for (int j = 0; j < SE_L_PER; ++j) {
    const int l = l0 + warp + 8 * j;
    if (l >= n_band) continue;
#pragma unroll
    for (int t = 0; t < SE_T_TILE; ++t) {
      if (t >= t_here) break;
      work[(((size_t)blockIdx.x * n_t + t0 + t) * n_band + l) * n_freq + f] = scale * acc[j][t];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Wigner coherence conductivity (DESIGN.md section 12.10).  Per q of the call and Cartesian axis a, with E[k][s] =
// eigvecs[q][s][k] (mode-major) and c^2 = THZ_PER_SQRT_EV_A2_AMU^2, the velocity operator (THz A)
//   W_a = dD/dQ_a E,   V_a[s][s'] = c^2 (E^H W_a)[s][s'] / (|nu_s| + |nu_s'|)   (0 where both are 0)
// by two batched complex GEMMs (coh_gemm_kernel, STAGE 0 then 1; W and V live in scratch only).  coh_pair_kernel:
// block (range of q, tile of COH_T_TILE temperatures); each thread owns (s, s') pairs of one q at a time and adds, for
// every ordered pair of modes kept (nu >= cutoff, Gamma > 0) in different degenerate sets (set_id),
//   (nu_s + nu_s') / 4 (C_s / nu_s + C_s' / nu_s') Re(V_a[s][s'] conj(V_b[s][s'])) L,
//   L = (Gamma_s + Gamma_s') / (2 pi [(nu_s - nu_s')^2 + (Gamma_s + Gamma_s')^2]),
// for the 6 components (a, b) and the tile's temperatures in registers.  V is Hermitian, so conj(V_b[s][s']) stands for
// V_b[s'][s] and every term is symmetric in (a, b).  The block reduces in a fixed order (warp shuffles, then the warps
// in order) and writes work[chunk][t][6]; chunk_reduce_kernel adds the chunks in chunk order into kappa [t][3][3].
// No atomics.
constexpr int COH_TILE = 32;   // GEMM output tile (both dimensions)
constexpr int COH_KTILE = 16;  // GEMM reduction tile
constexpr int COH_THREADS = 256;
constexpr int COH_T_TILE = 4;  // temperatures per pair block

// STAGE 0: out[q][a] = W_a [k][s'] = sum_k' ddyn[q][a][k][k'] E[k'][s'] (in = ddyn).  STAGE 1: out[q][a] = V_a [s][s']
// = c2 sum_k conj(E[k][s]) W_a[k][s'] / (|nu_s| + |nu_s'|) (in = W).  Grid (tiles of the [nb][nb] output, q, a).
template <int STAGE>
__global__ void __launch_bounds__(256)
coh_gemm_kernel(const double2* __restrict__ eig, const double2* __restrict__ in, const double* __restrict__ freqs, int nb,
                double c2, double2* __restrict__ out) {
  __shared__ double2 sa[COH_KTILE][COH_TILE];
  __shared__ double2 sb[COH_KTILE][COH_TILE + 1];
  const size_t nb2 = (size_t)nb * nb;
  const int q = blockIdx.y;
  const int tn = (nb + COH_TILE - 1) / COH_TILE;
  const int m0 = blockIdx.x / tn * COH_TILE, c0 = blockIdx.x % tn * COH_TILE;
  const double2* e = eig + (size_t)q * nb2;
  const double2* x = in + ((size_t)q * 3 + blockIdx.z) * nb2;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  double cr[2][2] = {{0.0, 0.0}, {0.0, 0.0}}, ci[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
  for (int k0 = 0; k0 < nb; k0 += COH_KTILE) {
    __syncthreads();  // the previous tiles have been read
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = threadIdx.x + 256 * r;
      const int am = i / COH_KTILE, ak = i % COH_KTILE;  // A(m0 + am, k0 + ak), row-major, k fastest
      double2 va = make_double2(0.0, 0.0);
      if (m0 + am < nb && k0 + ak < nb) {
        if constexpr (STAGE == 0) {
          va = __ldg(x + (size_t)(m0 + am) * nb + k0 + ak);
        } else {  // A(s, k) = conj(E[k][s]) = conj(eig[s][k])
          va = __ldg(e + (size_t)(m0 + am) * nb + k0 + ak);
          va.y = -va.y;
        }
      }
      sa[ak][am] = va;
      double2 vb = make_double2(0.0, 0.0);
      if constexpr (STAGE == 0) {  // B(k, n) = E[k][n] = eig[n][k]: k fastest
        const int bn = i / COH_KTILE, bk = i % COH_KTILE;
        if (c0 + bn < nb && k0 + bk < nb) vb = __ldg(e + (size_t)(c0 + bn) * nb + k0 + bk);
        sb[bk][bn] = vb;
      } else {  // B(k, n) = W[k][n], row-major
        const int bk = i / COH_TILE, bn = i % COH_TILE;
        if (c0 + bn < nb && k0 + bk < nb) vb = __ldg(x + (size_t)(k0 + bk) * nb + c0 + bn);
        sb[bk][bn] = vb;
      }
    }
    __syncthreads();
    const int kn = min(COH_KTILE, nb - k0);
    for (int kk = 0; kk < kn; ++kk) {
      const double2 a0 = sa[kk][ty], a1 = sa[kk][ty + 16];
      const double2 b0 = sb[kk][tx], b1 = sb[kk][tx + 16];
      cr[0][0] = fma(a0.x, b0.x, fma(-a0.y, b0.y, cr[0][0]));
      ci[0][0] = fma(a0.x, b0.y, fma(a0.y, b0.x, ci[0][0]));
      cr[0][1] = fma(a0.x, b1.x, fma(-a0.y, b1.y, cr[0][1]));
      ci[0][1] = fma(a0.x, b1.y, fma(a0.y, b1.x, ci[0][1]));
      cr[1][0] = fma(a1.x, b0.x, fma(-a1.y, b0.y, cr[1][0]));
      ci[1][0] = fma(a1.x, b0.y, fma(a1.y, b0.x, ci[1][0]));
      cr[1][1] = fma(a1.x, b1.x, fma(-a1.y, b1.y, cr[1][1]));
      ci[1][1] = fma(a1.x, b1.y, fma(a1.y, b1.x, ci[1][1]));
    }
  }
  double2* o = out + ((size_t)q * 3 + blockIdx.z) * nb2;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int m = m0 + ty + 16 * i, c = c0 + tx + 16 * j;
      if (m >= nb || c >= nb) continue;
      if constexpr (STAGE == 0) {
        o[(size_t)m * nb + c] = make_double2(cr[i][j], ci[i][j]);
      } else {
        const double den = fabs(__ldg(freqs + (size_t)q * nb + m)) + fabs(__ldg(freqs + (size_t)q * nb + c));
        o[(size_t)m * nb + c] = den > 0.0 ? make_double2(c2 * cr[i][j] / den, c2 * ci[i][j] / den)
                                          : make_double2(0.0, 0.0);
      }
    }
  }
}

__global__ void __launch_bounds__(COH_THREADS)
coh_pair_kernel(const double* __restrict__ freqs, const int32_t* __restrict__ set_id, const double2* __restrict__ vel,
                const double* __restrict__ cv, const double* __restrict__ gamma, int n_q, int nb, int n_t,
                double cutoff, double* __restrict__ work) {
  __shared__ double red[COH_THREADS / 32][6 * COH_T_TILE];
  const int t0 = blockIdx.y * COH_T_TILE;
  const int t_here = min(COH_T_TILE, n_t - t0);
  const int q_begin = (int)((int64_t)n_q * blockIdx.x / gridDim.x);
  const int q_end = (int)((int64_t)n_q * (blockIdx.x + 1) / gridDim.x);
  const int64_t nb2 = (int64_t)nb * nb;
  double acc[6][COH_T_TILE];
#pragma unroll
  for (int c = 0; c < 6; ++c)
#pragma unroll
    for (int t = 0; t < COH_T_TILE; ++t) acc[c][t] = 0.0;
  for (int q = q_begin; q < q_end; ++q) {
    const double* nu = freqs + (size_t)q * nb;
    const int32_t* sid = set_id + (size_t)q * nb;
    const double2* v = vel + (size_t)q * 3 * nb2;
    for (int64_t i = threadIdx.x; i < nb2; i += COH_THREADS) {
      const int s = (int)(i / nb), sp = (int)(i % nb);
      const double n1 = __ldg(nu + s), n2 = __ldg(nu + sp);
      if (!(n1 >= cutoff && n2 >= cutoff) || __ldg(sid + s) == __ldg(sid + sp)) continue;
      const double2 vx = __ldg(v + i), vy = __ldg(v + nb2 + i), vz = __ldg(v + 2 * nb2 + i);
      double prod[6];  // Re(V_a conj(V_b)) in Voigt order xx, yy, zz, yz, xz, xy
      prod[0] = fma(vx.x, vx.x, vx.y * vx.y);
      prod[1] = fma(vy.x, vy.x, vy.y * vy.y);
      prod[2] = fma(vz.x, vz.x, vz.y * vz.y);
      prod[3] = fma(vy.x, vz.x, vy.y * vz.y);
      prod[4] = fma(vx.x, vz.x, vx.y * vz.y);
      prod[5] = fma(vx.x, vy.x, vx.y * vy.y);
      const double quarter = 0.25 * (n1 + n2), dnu = n1 - n2;
#pragma unroll
      for (int t = 0; t < COH_T_TILE; ++t) {
        if (t >= t_here) break;
        const size_t o = ((size_t)(t0 + t) * n_q + q) * nb;
        const double g1 = __ldg(gamma + o + s), g2 = __ldg(gamma + o + sp);
        if (!(g1 > 0.0 && g2 > 0.0)) continue;
        const double gs = g1 + g2;
        const double w = quarter * (__ldg(cv + o + s) / n1 + __ldg(cv + o + sp) / n2) * gs /
                         (2.0 * 3.141592653589793 * fma(dnu, dnu, gs * gs));
#pragma unroll
        for (int c = 0; c < 6; ++c) acc[c][t] = fma(w, prod[c], acc[c][t]);
      }
    }
  }
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
#pragma unroll
  for (int c = 0; c < 6; ++c) {
#pragma unroll
    for (int t = 0; t < COH_T_TILE; ++t) {
      double x = acc[c][t];
#pragma unroll
      for (int off = 16; off > 0; off /= 2) x += __shfl_down_sync(0xffffffffu, x, off);
      if (lane == 0) red[warp][t * 6 + c] = x;
    }
  }
  __syncthreads();
  if (threadIdx.x < 6 * t_here) {
    double s = 0.0;
    for (int w = 0; w < COH_THREADS / 32; ++w) s += red[w][threadIdx.x];
    work[((size_t)blockIdx.x * n_t + t0) * 6 + threadIdx.x] = s;
  }
}

struct SymmetricStore {  // work[chunk][t][6] (xx, yy, zz, yz, xz, xy): kappa[t][a][b] and kappa[t][b][a] += the sum
  double* kappa;
  __device__ void operator()(int64_t o, double s) const {
    const int c = (int)(o % 6);
    const int a = c < 3 ? c : (c == 3 ? 1 : 0), b = c < 3 ? c : (c == 5 ? 1 : 2);
    double* k = kappa + (o / 6) * 9;
    k[a * 3 + b] += s;
    if (a != b) k[b * 3 + a] += s;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// Isotope scattering (DESIGN.md section 12.11).  For target t of the call (mesh index targets[t]) and band l at the
// frequency w = omega[t][l]:
//   gamma[t][l] = (pi / 4) w^2 (1 / 6N) sum over the tetrahedra T of the mesh and the bands l' of
//                 sum_v wt_v(w; T, l') O[t][q_v][l'][l],
//   O[t][q'][l'][l] = sum_k g_k |sum_a conj(e_ka(t, l)) e_ka(q', l')|^2   (0 where freqs[q'][l'] < cutoff),
// wt_v tetra_weights' corner weight of corner q_v for the corner values freqs[q_v][l'].  Summed per tetrahedron this is
// (1/N) sum_q' W_l'(q'; w) O with W the vertex weight 1/6 sum over the 24 (tetrahedron, corner) at q'.  Gamma = 0 where
// w < cutoff.  iso_overlap_kernel: one thread per element of O [t][q'][l'][l], l fastest.  iso_accumulate_kernel:
// block (chunk of (tetrahedron, l') items, band tile, target); each tile of items is sorted into shared memory as in
// tetrahedron_dos_kernel, then thread (slice s, band l) adds the items s, s + S, ... of the tile at its own w, reading
// O coalesced along l; the slices are added in order in shared memory and the block writes work[chunk][t][l].
// chunk_reduce_kernel adds the chunks in chunk order and applies (pi / 4) w^2 / 6N.  The chunks depend on the mesh and
// the band count only, so a target's result does not depend on the other targets of the call.  No atomics.
constexpr int ISO_THREADS = 256;  // threads per block, and items staged per tile

__global__ void __launch_bounds__(ISO_THREADS)
iso_overlap_kernel(const double2* __restrict__ eig, const double* __restrict__ freqs, int n_band, int n_q,
                   const double* __restrict__ g, int n_prim, const int32_t* __restrict__ targets, int n_target,
                   double cutoff, double* __restrict__ overlap) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t nb2 = (int64_t)n_band * n_band, per_t = (int64_t)n_q * nb2;
  if (i >= (int64_t)n_target * per_t) return;
  const int t = (int)(i / per_t), q = (int)((i / nb2) % n_q), lp = (int)((i / n_band) % n_band);
  const int l = (int)(i % n_band);
  double o = 0.0;
  if (__ldg(freqs + (size_t)q * n_band + lp) >= cutoff) {
    const double2* a = eig + ((size_t)__ldg(targets + t) * n_band + l) * n_band;
    const double2* b = eig + ((size_t)q * n_band + lp) * n_band;
    for (int k = 0; k < n_prim; ++k) {
      double re = 0.0, im = 0.0;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double2 x = __ldg(a + 3 * k + c), y = __ldg(b + 3 * k + c);
        re = fma(x.x, y.x, fma(x.y, y.y, re));
        im = fma(x.x, y.y, fma(-x.y, y.x, im));
      }
      o = fma(__ldg(g + k), fma(re, re, im * im), o);
    }
  }
  overlap[i] = o;
}

__global__ void __launch_bounds__(ISO_THREADS)
iso_accumulate_kernel(const double* __restrict__ freqs, int n_band, int n1, int n2, int n3,
                      const int32_t* __restrict__ tet, const double* __restrict__ omega,
                      const double* __restrict__ overlap, int n_target, int l_tile, double cutoff,
                      double* __restrict__ work) {
  __shared__ double se[ISO_THREADS][4];
  __shared__ int32_t sq[ISO_THREADS][4];
  __shared__ int32_t sb[ISO_THREADS];
  __shared__ double red[ISO_THREADS];
  const int t = blockIdx.z;
  const int n_slices = ISO_THREADS / l_tile;
  const int s = threadIdx.x / l_tile, l = blockIdx.y * l_tile + threadIdx.x % l_tile;
  const bool active = s < n_slices && l < n_band;
  const double w = active ? __ldg(omega + (size_t)t * n_band + l) : 0.0;
  const bool live = active && w >= cutoff;
  const int64_t n_q = (int64_t)n1 * n2 * n3, nb2 = (int64_t)n_band * n_band;
  const double* o_t = overlap + (size_t)t * n_q * nb2 + l;
  const int64_t n_items = n_q * 6 * n_band;
  const int64_t n_tiles = (n_items + ISO_THREADS - 1) / ISO_THREADS;
  const int64_t t_end = n_tiles * (blockIdx.x + 1) / gridDim.x;
  double acc = 0.0;
  for (int64_t tile = n_tiles * blockIdx.x / gridDim.x; tile < t_end; ++tile) {
    const int64_t p = tile * ISO_THREADS + threadIdx.x;
    __syncthreads();  // the previous tile has been read
    if (p < n_items) {
      const int band = (int)(p % n_band);
      double e[4];
      int32_t q[4];
      tetrahedron_corners(tet, p / n_band, n1, n2, n3, [&](int v, int a, int b, int c) {
        q[v] = (a * n2 + b) * n3 + c;
        e[v] = __ldg(freqs + (int64_t)q[v] * n_band + band);
      });
      sort4(e, q);
#pragma unroll
      for (int v = 0; v < 4; ++v) se[threadIdx.x][v] = e[v], sq[threadIdx.x][v] = q[v];
      sb[threadIdx.x] = band;
    }
    __syncthreads();
    if (!live) continue;
    const int n_here = (int)min((int64_t)ISO_THREADS, n_items - tile * ISO_THREADS);
    for (int i = s; i < n_here; i += n_slices) {
      const double e[4] = {se[i][0], se[i][1], se[i][2], se[i][3]};
      if (!(w >= e[0] && w < e[3])) continue;
      double n, gw, wt[4];
      tetra_weights(w, e, n, gw, wt);
      const int64_t lp = sb[i];
#pragma unroll
      for (int v = 0; v < 4; ++v) acc = fma(wt[v], __ldg(o_t + (sq[i][v] * n_band + lp) * n_band), acc);
    }
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  if (active && s == 0) {
    double sum = 0.0;
    for (int k = 0; k < n_slices; ++k) sum += red[k * l_tile + threadIdx.x];
    work[((size_t)blockIdx.x * n_target + t) * n_band + l] = sum;
  }
}

struct IsotopeStore {  // work[chunk][t][l]: gamma[t][l] = scale * omega[t][l]^2 * the sum
  double* gamma;
  const double* omega;
  double scale;
  __device__ void operator()(int64_t o, double s) const {
    const double w = omega[o];
    gamma[o] = s * (scale * w * w);
  }
};

// ---------------------------------------------------------------------------------------------------------------
// Effective force constants by stochastic sampling (DESIGN.md section 12.12).
//
// chg_sample_displacements, three stages: eff_variates_kernel writes xi[s][lam] = amp[lam] xi(seed, iteration,
// first_sample + s, lam), the standard normal of a splitmix64 hash of the counter by Box-Muller, so a sample does not
// depend on how the samples are split over calls; eff_superpose_kernel is the fp64 product d[s][i] = inv_sqrt_m[i / 3]
// sum_lam xi[s][lam] E[lam][i] (64 x 64 output tiles, lam ascending, one thread 4 x 4 outputs); eff_positions_kernel
// turns each atom's draw into fp32 fractional coordinates and writes the fp64 displacement the model sees,
// u = (frac32 - fp32(frac_ref)) L.
//
// chg_displacement_moments: eff_moments_kernel, one thread per (sample, primitive atom kappa, supercell atom j), sums
// over the n_cells translations l in order and writes the sample's partial sums of G_c and B for (kappa, j) to work
// slot 1 + s; the thread (s, 0, 0) also writes the sample's |dF|^2 and F_0 . u; the threads of sample 0 copy the running
// sums acc into slot 0.  chunk_reduce_kernel then adds the slots in order, acc = (((acc + p_0) + p_1) + ...): a left fold
// over the samples in order, so the result is bitwise independent of how the samples are split over calls.  No atomics.
constexpr int EFF_THREADS = 256;
constexpr int EFF_TILE = 64;  // output tile of eff_superpose_kernel (samples x coordinates)
constexpr int EFF_BK = 16;    // modes staged per step

__device__ __forceinline__ uint64_t eff_mix(uint64_t x) {  // splitmix64
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__global__ void __launch_bounds__(EFF_THREADS)
eff_variates_kernel(const double* __restrict__ amp, int n_modes, uint64_t seed, uint64_t iteration,
                    uint64_t first_sample, int n_samples, double* __restrict__ xi) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_samples * n_modes) return;
  const uint64_t s = first_sample + (uint64_t)(i / n_modes), lam = (uint64_t)(i % n_modes);
  const uint64_t r = eff_mix(eff_mix(eff_mix(eff_mix(seed) + iteration) + s) + lam);
  const double u1 = (double)((r >> 11) + 1) * 0x1.0p-53;  // (0, 1]
  const double u2 = (double)(eff_mix(r) >> 11) * 0x1.0p-53;  // [0, 1)
  xi[i] = __ldg(amp + lam) * (sqrt(-2.0 * log(u1)) * cospi(2.0 * u2));
}

__global__ void __launch_bounds__(EFF_THREADS)
eff_superpose_kernel(const double* __restrict__ xi, const double* __restrict__ evecs,
                     const double* __restrict__ inv_sqrt_m, int n_samples, int n_modes, double* __restrict__ d) {
  __shared__ double sa[EFF_BK][EFF_TILE + 1];  // sa[lam][s]
  __shared__ double sb[EFF_BK][EFF_TILE];      // sb[lam][i]
  const int s0 = blockIdx.y * EFF_TILE, i0 = blockIdx.x * EFF_TILE;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  double acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
  for (int k0 = 0; k0 < n_modes; k0 += EFF_BK) {
    for (int e = threadIdx.x; e < EFF_BK * EFF_TILE; e += EFF_THREADS) {
      const int r = e / EFF_BK, ka = e % EFF_BK;  // xi read along lam
      const int s = s0 + r, la = k0 + ka;
      sa[ka][r] = (s < n_samples && la < n_modes) ? __ldg(xi + (size_t)s * n_modes + la) : 0.0;
      const int kb = e / EFF_TILE, c = e % EFF_TILE;  // E read along i
      const int lb = k0 + kb, i = i0 + c;
      sb[kb][c] = (lb < n_modes && i < n_modes) ? __ldg(evecs + (size_t)lb * n_modes + i) : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < EFF_BK; ++k) {
      double a[4], b[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) a[r] = sa[k][ty + 16 * r];
#pragma unroll
      for (int c = 0; c < 4; ++c) b[c] = sb[k][tx + 16 * c];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = fma(a[r], b[c], acc[r][c]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int s = s0 + ty + 16 * r;
    if (s >= n_samples) continue;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int i = i0 + tx + 16 * c;
      if (i < n_modes) d[(size_t)s * n_modes + i] = acc[r][c] * __ldg(inv_sqrt_m + i / 3);
    }
  }
}

// u [s][a] holds the fp64 draw d on entry and the displacement the model sees on exit
__global__ void __launch_bounds__(EFF_THREADS)
eff_positions_kernel(const double* __restrict__ frac_ref, const double* __restrict__ lattice,
                     const double* __restrict__ inv_lattice, int n_atoms, int n_samples, float* __restrict__ frac,
                     double* __restrict__ u) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_samples * n_atoms) return;
  const int a = (int)(i % n_atoms);
  double* ui = u + (size_t)i * 3;
  const double d[3] = {ui[0], ui[1], ui[2]};
  double du[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double ref = __ldg(frac_ref + (size_t)a * 3 + c);
    const double x = ref + (d[0] * __ldg(inv_lattice + c) + d[1] * __ldg(inv_lattice + 3 + c) +
                            d[2] * __ldg(inv_lattice + 6 + c));
    const float x32 = __double2float_rn(x);
    frac[(size_t)i * 3 + c] = x32;
    du[c] = (double)x32 - (double)__double2float_rn(ref);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c)
    ui[c] = du[0] * __ldg(lattice + c) + du[1] * __ldg(lattice + 3 + c) + du[2] * __ldg(lattice + 6 + c);
}

__global__ void __launch_bounds__(EFF_THREADS)
eff_moments_kernel(const double* __restrict__ u, const double* __restrict__ force, const double* __restrict__ f0,
                   const int32_t* __restrict__ perm, int n_atoms, int n_cells, int n_prim,
                   const double* __restrict__ acc, double* __restrict__ work) {
  const int64_t n_g = (int64_t)n_prim * 9 * n_atoms, n_out = 2 * n_g + 2;
  const int s = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;  // kappa n_atoms + j
  const double* us = u + (size_t)s * n_atoms * 3;
  const double* fs = force + (size_t)s * n_atoms * 3;
  double* w = work + (size_t)(s + 1) * n_out;
  if (t < n_prim * n_atoms) {
    const int k = t / n_atoms, j = t % n_atoms;
    double g[9], b[9];
#pragma unroll
    for (int x = 0; x < 9; ++x) g[x] = b[x] = 0.0;
    for (int l = 0; l < n_cells; ++l) {
      const int a = __ldg(perm + (size_t)l * n_atoms + k * n_cells), c = __ldg(perm + (size_t)l * n_atoms + j);
      double ua[3], df[3], uc[3];
#pragma unroll
      for (int x = 0; x < 3; ++x) {
        ua[x] = __ldg(us + a * 3 + x);
        df[x] = __ldg(fs + a * 3 + x) - __ldg(f0 + a * 3 + x);
        uc[x] = __ldg(us + c * 3 + x);
      }
#pragma unroll
      for (int x = 0; x < 3; ++x)
#pragma unroll
        for (int y = 0; y < 3; ++y) {
          g[3 * x + y] = fma(ua[x], uc[y], g[3 * x + y]);
          b[3 * x + y] = fma(df[x], uc[y], b[3 * x + y]);
        }
    }
#pragma unroll
    for (int x = 0; x < 3; ++x)
#pragma unroll
      for (int y = 0; y < 3; ++y) {
        const int64_t o = ((int64_t)(k * 3 + x) * n_atoms + j) * 3 + y;
        w[o] = g[3 * x + y];
        w[n_g + o] = b[3 * x + y];
        if (s == 0) work[o] = acc[o], work[n_g + o] = acc[n_g + o];
      }
  }
  if (t == 0) {
    double ss = 0.0, wf = 0.0;
    for (int i = 0; i < 3 * n_atoms; ++i) {
      const double f = __ldg(f0 + i), df = __ldg(fs + i) - f;
      ss = fma(df, df, ss);
      wf = fma(f, __ldg(us + i), wf);
    }
    w[2 * n_g] = ss;
    w[2 * n_g + 1] = wf;
    if (s == 0) work[2 * n_g] = acc[2 * n_g], work[2 * n_g + 1] = acc[2 * n_g + 1];
  }
}

struct CopyStore {  // out[o] = the sum
  double* out;
  __device__ void operator()(int64_t o, double s) const { out[o] = s; }
};

}  // namespace
}  // namespace chg

using namespace chg;

#define CHG_DYN_CHECKS()                                                                     \
  CHG_CHECK_ARG(n_prim >= 0 && n_super >= 0 && n_q >= 0, "negative size");                   \
  if (n_prim == 0 || n_q == 0) return CHG_OK;                                                \
  CHG_CHECK_ARG(fc && img_ptr && img_vec && s2p && inv_sqrt_m && qpoints && dyn, "null pointer"); \
  CHG_CHECK_ARG((int64_t)n_prim * n_prim < (1ll << 31), "too many primitive atoms");         \
  const int64_t q_blocks = ((int64_t)n_q + DYN_THREADS - 1) / DYN_THREADS;                    \
  CHG_CHECK_ARG(q_blocks <= 65535, "too many q-points in one call (at most 65535 * 128)")

extern "C" int chg_dynamical_matrices(const double* fc, const int32_t* img_ptr, const double* img_vec,
                                      const int32_t* s2p, const double* inv_sqrt_m, int32_t n_prim, int32_t n_super,
                                      const double* qpoints, int32_t n_q, double* dyn, void* stream) {
  CHG_DYN_CHECKS();
  const dim3 grid((unsigned)(n_prim * n_prim), (unsigned)q_blocks);
  dynamical_matrices_kernel<false><<<grid, DYN_THREADS, 0, as_stream(stream)>>>(
      fc, img_ptr, img_vec, s2p, inv_sqrt_m, n_prim, n_super, qpoints, n_q, nullptr, dyn);
  CHG_LAUNCH_END();
}

extern "C" int chg_dynamical_matrix_derivatives(const double* fc, const int32_t* img_ptr, const double* img_vec,
                                                const int32_t* s2p, const double* inv_sqrt_m, int32_t n_prim,
                                                int32_t n_super, const double* qpoints, int32_t n_q,
                                                const double* prim_lattice, double* dyn, void* stream) {
  CHG_DYN_CHECKS();
  CHG_CHECK_ARG(prim_lattice, "null pointer");
  const dim3 grid((unsigned)(n_prim * n_prim), (unsigned)q_blocks, 3);
  dynamical_matrices_kernel<true><<<grid, DYN_THREADS, 0, as_stream(stream)>>>(
      fc, img_ptr, img_vec, s2p, inv_sqrt_m, n_prim, n_super, qpoints, n_q, prim_lattice, dyn);
  CHG_LAUNCH_END();
}
#undef CHG_DYN_CHECKS

extern "C" int chg_tetrahedron_dos(const double* freqs, int32_t n_band, int32_t n1, int32_t n2, int32_t n3,
                                   const int32_t* tetrahedra, const double* proj, int32_t n_proj,
                                   const double* omega, int32_t n_freq, double* dos, double* idos, double* pdos,
                                   double* work, void* stream) {
  CHG_CHECK_ARG(n_band >= 0 && n1 > 0 && n2 > 0 && n3 > 0 && n_freq >= 0 && n_proj >= 0, "bad size");
  CHG_CHECK_ARG((int64_t)n1 * n2 * n3 < (1ll << 31), "mesh too large");
  if (n_freq == 0) return CHG_OK;
  CHG_CHECK_ARG(freqs && tetrahedra && omega && dos && idos && work, "null pointer");
  CHG_CHECK_ARG(!proj || (pdos && n_proj > 0), "projections need pdos and n_proj > 0");
  const int64_t n_pairs = (int64_t)n1 * n2 * n3 * 6 * n_band;
  const int threads = (int)std::min<int64_t>(DOS_MAX_THREADS, ((int64_t)n_freq + 31) / 32 * 32);
  const int64_t f_blocks = ((int64_t)n_freq + threads - 1) / threads;
  const int64_t n_tiles = (n_pairs + threads - 1) / threads;
  const int chunks = (int)std::max<int64_t>(1, std::min<int64_t>(CHG_DOS_MAX_CHUNKS, n_tiles));
  const int groups = proj ? (n_proj + DOS_PROJ - 1) / DOS_PROJ : 1;
  CHG_CHECK_ARG(f_blocks <= 65535 && groups <= 65535, "too many frequency points or projections");
  const int rows = 2 + (proj ? n_proj : 0);
  tetrahedron_dos_kernel<<<dim3(chunks, (unsigned)f_blocks, groups), threads, 0, as_stream(stream)>>>(
      freqs, n_band, n1, n2, n3, tetrahedra, proj, n_proj, omega, n_freq, n_pairs, work);
  const double scale = 1.0 / (6.0 * (double)n1 * n2 * n3);
  CHG_CUDA(reduce_chunks(work, chunks, (int64_t)rows * n_freq, DosStore{dos, idos, pdos, n_freq, scale},
                         as_stream(stream)));
  CHG_LAUNCH_END();
}

extern "C" int chg_thermal_displacements(const double* freqs, const double* eigvecs, int32_t n_q, int32_t n_prim,
                                         const double* temperatures, int32_t n_t, double cutoff_thz, double* work,
                                         double* acc, void* stream) {
  CHG_CHECK_ARG(n_q >= 0 && n_prim >= 0 && n_t >= 0, "negative size");
  if (n_q == 0 || n_prim == 0 || n_t == 0) return CHG_OK;
  CHG_CHECK_ARG(freqs && eigvecs && temperatures && work && acc, "null pointer");
  const int64_t groups = ((int64_t)n_prim + TD_ATOMS - 1) / TD_ATOMS;
  const int64_t t_tiles = ((int64_t)n_t + TD_THREADS - 1) / TD_THREADS;
  CHG_CHECK_ARG(groups <= 65535 && t_tiles <= 65535, "too many atoms or temperatures");
  const int t_tile = (int)((n_t + t_tiles - 1) / t_tiles);
  const int n_qi = TD_THREADS / t_tile;
  const int chunks = (int)std::min<int64_t>(CHG_TD_MAX_CHUNKS, ((int64_t)n_q + n_qi - 1) / n_qi);
  thermal_displacements_kernel<<<dim3(chunks, (unsigned)groups, (unsigned)t_tiles), n_qi * t_tile, 0,
                                 as_stream(stream)>>>(freqs, reinterpret_cast<const double2*>(eigvecs), n_q, n_prim,
                                                      temperatures, n_t, t_tile, cutoff_thz, work);
  CHG_CUDA(reduce_chunks(work, chunks, (int64_t)n_t * n_prim * 6, AccumulateStore{acc}, as_stream(stream)));
  CHG_LAUNCH_END();
}

extern "C" int chg_joint_dos(const double* freqs, int32_t n_band, int32_t n1, int32_t n2, int32_t n3,
                             const int32_t* tetrahedra, const int32_t* targets, int32_t n_target, const double* omega,
                             int32_t n_freq, const double* temperatures, int32_t n_t, double cutoff_thz, double* out,
                             double* work, void* stream) {
  CHG_CHECK_ARG(n_band >= 0 && n1 > 0 && n2 > 0 && n3 > 0 && n_target >= 0 && n_freq >= 0 && n_t >= 0, "bad size");
  CHG_CHECK_ARG((int64_t)n1 * n2 * n3 * std::max(n_band, 1) < (1ll << 31), "mesh too large");
  CHG_CHECK_ARG(n_t < 65535, "too many temperatures");
  if (n_target == 0 || n_freq == 0) return CHG_OK;
  CHG_CHECK_ARG(freqs && tetrahedra && targets && omega && out && work && (n_t == 0 || temperatures), "null pointer");
  const int64_t n_items = (int64_t)n1 * n2 * n3 * 6 * n_band * n_band;
  const int threads = (int)std::min<int64_t>(JDOS_THREADS, ((int64_t)n_freq + 31) / 32 * 32);
  const int per_block = JDOS_THREADS / threads;  // target slots per block
  const int64_t f_tiles = ((int64_t)n_freq + threads - 1) / threads;
  const int64_t groups = ((int64_t)n_target + per_block - 1) / per_block * f_tiles;
  CHG_CHECK_ARG(groups <= 65535, "too many targets or frequency points in one call");
  const int n_slots = 1 + n_t;
  // enough chunks for about 4 096 blocks in all, at most CHG_JDOS_MAX_CHUNKS and one tile each
  const int64_t n_tiles = (n_items + threads - 1) / threads;
  const int64_t want = (4096 + groups * n_slots - 1) / (groups * n_slots);
  const int chunks = (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)CHG_JDOS_MAX_CHUNKS, n_tiles, want}));
  joint_dos_kernel<<<dim3(chunks, (unsigned)groups, n_slots), dim3(threads, per_block), 0, as_stream(stream)>>>(
      freqs, n_band, n1, n2, n3, tetrahedra, targets, n_target, omega, n_freq, temperatures, cutoff_thz,
      n_items, work);
  const double scale = 1.0 / (6.0 * (double)n1 * n2 * n3);
  CHG_CUDA(reduce_chunks(work, chunks, (int64_t)n_target * n_slots * 2 * n_freq, JointDosStore{out, n_freq, scale},
                         as_stream(stream)));
  CHG_LAUNCH_END();
}

extern "C" int chg_structure_factors(const double* freqs, const double* eigvecs, const double* kcart,
                                     const double* gvec, const double* frac, const double* coef, const double* u,
                                     const double* temperatures, int32_t n_t, int32_t n_q, int32_t n_prim,
                                     double cutoff_thz, double* out, void* stream) {
  CHG_CHECK_ARG(n_t >= 0 && n_q >= 0 && n_prim >= 0, "negative size");
  if (n_t == 0 || n_q == 0 || n_prim == 0) return CHG_OK;
  CHG_CHECK_ARG(freqs && eigvecs && kcart && gvec && frac && coef && temperatures && out, "null pointer");
  const int64_t n_items = (int64_t)n_q * 3 * n_prim;
  const int64_t blocks = (n_items + SQW_THREADS - 1) / SQW_THREADS;
  const int64_t t_tiles = u ? ((int64_t)n_t + SQW_T_TILE - 1) / SQW_T_TILE : 1;
  CHG_CHECK_ARG(blocks < (1ll << 31) && t_tiles <= 65535, "too many rows or temperatures in one call");
  structure_factors_kernel<<<dim3((unsigned)blocks, (unsigned)t_tiles), SQW_THREADS, 0, as_stream(stream)>>>(
      freqs, reinterpret_cast<const double2*>(eigvecs), kcart, gvec, frac, coef, u, temperatures, n_t, n_q, n_prim,
      cutoff_thz, out);
  CHG_LAUNCH_END();
}

extern "C" int chg_broadened_spectrum(const double* freqs, const double* weights, int32_t n_q, int32_t n_modes,
                                      int32_t n_t, int64_t row0, int32_t group_size, int64_t n_groups,
                                      const double* omega, int32_t n_freq, double sigma, double* work,
                                      int64_t work_doubles, double* out, void* stream) {
  CHG_CHECK_ARG(n_q >= 0 && n_modes >= 0 && n_t >= 0 && n_freq >= 0 && row0 >= 0 && group_size > 0, "bad size");
  if (n_q == 0 || n_modes == 0 || n_t == 0 || n_freq == 0) return CHG_OK;
  CHG_CHECK_ARG(freqs && weights && omega && work && out, "null pointer");
  CHG_CHECK_ARG(sigma > 0.0, "sigma must be positive");
  const int64_t g_first = row0 / group_size, g_last = (row0 + n_q - 1) / group_size;
  CHG_CHECK_ARG(g_last < n_groups, "rows beyond the last group");
  const int n_groups_here = (int)(g_last - g_first + 1);
  const int threads = (int)std::min<int64_t>(SQW_BROAD_THREADS, ((int64_t)n_freq + 31) / 32 * 32);
  const int64_t f_blocks = ((int64_t)n_freq + threads - 1) / threads;
  CHG_CHECK_ARG(f_blocks <= 65535, "too many frequency points in one call");
  // scratch of one chunk: every (t, group, f) of the call
  const int64_t per_chunk = (int64_t)n_t * n_groups_here * n_freq;
  CHG_CHECK_ARG(work_doubles >= per_chunk, "work holds less than one chunk (n_t x groups in the call x n_freq)");
  // enough chunks for about 4 096 blocks in all, at most CHG_SQW_MAX_CHUNKS, one tile of the largest group each, and
  // no more than work holds
  const int64_t most = (int64_t)std::min(group_size, n_q) * n_modes;
  const int64_t n_tiles = (most + threads - 1) / threads;
  const int64_t others = f_blocks * n_groups_here * n_t;
  const int64_t want = (4096 + others - 1) / others;
  const int chunks = (int)std::max<int64_t>(
      1, std::min<int64_t>({(int64_t)CHG_SQW_MAX_CHUNKS, n_tiles, want, work_doubles / per_chunk}));
  const int64_t x_blocks = (int64_t)chunks * n_groups_here * n_t;
  CHG_CHECK_ARG(x_blocks < (1ll << 31), "too many groups or temperatures in one call");
  broadened_spectrum_kernel<<<dim3((unsigned)x_blocks, (unsigned)f_blocks), threads, 0, as_stream(stream)>>>(
      freqs, reinterpret_cast<const double2*>(weights), n_q, n_modes, n_t, row0, group_size, n_groups_here, omega,
      n_freq, sigma, chunks, work);
  CHG_CUDA(reduce_chunks(work, chunks, (int64_t)n_t * n_groups_here * n_freq,
                         SpectrumStore{out, n_freq, n_groups_here, g_first, n_groups, 1.0 / group_size},
                         as_stream(stream)));
  CHG_LAUNCH_END();
}

extern "C" int chg_phonon_interaction(const double* fc3, const int32_t* img_ptr, const double* img_vec,
                                      const int32_t* s2p, const double* inv_sqrt_m, const double* frac, int32_t n_prim,
                                      int32_t n_super, int32_t n1, int32_t n2, int32_t n3, const double* freqs,
                                      const double* eigvecs, int32_t target, const int32_t* q1_idx, int32_t n_q1,
                                      double cutoff_thz, double* work, int64_t work_doubles, double* out,
                                      void* stream) {
  CHG_CHECK_ARG(n_prim >= 0 && n_super >= 0 && n_q1 >= 0 && n1 > 0 && n2 > 0 && n3 > 0, "bad size");
  CHG_CHECK_ARG((int64_t)n1 * n2 * n3 < (1ll << 31), "mesh too large");
  CHG_CHECK_ARG(target >= 0 && (int64_t)target < (int64_t)n1 * n2 * n3, "target outside the mesh");
  if (n_prim == 0 || n_q1 == 0) return CHG_OK;
  CHG_CHECK_ARG(fc3 && img_ptr && img_vec && s2p && inv_sqrt_m && frac && freqs && eigvecs && q1_idx && work && out,
                "null pointer");
  CHG_CHECK_ARG(n_super % n_prim == 0, "n_super must be a multiple of n_prim (atom-major supercell)");
  CHG_CHECK_ARG(n_q1 <= 65535, "too many q1 in one call (at most 65535)");
  const int64_t nb = 3 * (int64_t)n_prim, n33 = nb * nb * nb;
  const int64_t rho_n = (int64_t)n_q1 * 2 * n_prim * n_super;
  CHG_CHECK_ARG(work_doubles >= 2 * (rho_n + 2 * (int64_t)n_q1 * n33), "work holds less than 4 n_q1 (n_prim n_super + (3 n_prim)^3) doubles");
  double2* rho = reinterpret_cast<double2*>(work);
  double2* buf_a = rho + rho_n;
  double2* buf_b = buf_a + (size_t)n_q1 * n33;
  const double2* eig = reinterpret_cast<const double2*>(eigvecs);
  cudaStream_t st = as_stream(stream);
  rho_kernel<<<(unsigned)((rho_n + PH3_THREADS - 1) / PH3_THREADS), PH3_THREADS, 0, st>>>(
      img_ptr, img_vec, s2p, inv_sqrt_m, frac, n_prim, n_super, n1, n2, n3, target, q1_idx, n_q1, rho);
  count_launch();
  const int64_t n_r = (int64_t)n_prim * n_prim * n_prim * 27;
  const dim3 rgrid((unsigned)((n_r + PH3_THREADS - 1) / PH3_THREADS), (unsigned)((n_q1 + PH3_Q1_TILE - 1) / PH3_Q1_TILE));
  fc3_fourier_kernel<<<rgrid, PH3_THREADS, 0, st>>>(fc3, rho, n_prim, n_super, n_q1, buf_a);
  count_launch();
  const int64_t t1 = (nb + PH3_TILE - 1) / PH3_TILE, t2 = (nb * nb + PH3_TILE - 1) / PH3_TILE;
  const double p_scale = SQW_C * SQW_C * SQW_C / (36.0 * (double)n1 * n2 * n3);
  contract_kernel<0><<<dim3((unsigned)(t1 * t2), 1, n_q1), 256, 0, st>>>(
      eig, freqs, n_prim, n1, n2, n3, target, q1_idx, cutoff_thz, p_scale, buf_a, buf_b, nullptr);
  count_launch();
  contract_kernel<1><<<dim3((unsigned)(nb * t1 * t1), 1, n_q1), 256, 0, st>>>(
      eig, freqs, n_prim, n1, n2, n3, target, q1_idx, cutoff_thz, p_scale, buf_b, buf_a, nullptr);
  count_launch();
  contract_kernel<2><<<dim3((unsigned)(t2 * t1), 1, n_q1), 256, 0, st>>>(
      eig, freqs, n_prim, n1, n2, n3, target, q1_idx, cutoff_thz, p_scale, buf_a, nullptr, out);
  CHG_LAUNCH_END();
}

extern "C" int chg_imag_self_energy(const double* freqs, int32_t n_band, int32_t n1, int32_t n2, int32_t n3,
                                    const int32_t* tetrahedra, int32_t target, const double* omega,
                                    const int32_t* q1_idx, int32_t n_q1, const double* p, const double* temperatures,
                                    int32_t n_t, double cutoff_thz, double* work, int64_t work_doubles, double* gamma,
                                    void* stream) {
  CHG_CHECK_ARG(n_band >= 0 && n1 > 0 && n2 > 0 && n3 > 0 && n_q1 >= 0 && n_t >= 0, "bad size");
  CHG_CHECK_ARG((int64_t)n1 * n2 * n3 * std::max(n_band, 1) < (1ll << 31), "mesh too large");
  CHG_CHECK_ARG(target >= 0 && (int64_t)target < (int64_t)n1 * n2 * n3, "target outside the mesh");
  if (n_band == 0 || n_q1 == 0 || n_t == 0) return CHG_OK;
  CHG_CHECK_ARG(freqs && tetrahedra && omega && q1_idx && p && temperatures && work && gamma, "null pointer");
  const int64_t nb2 = (int64_t)n_band * n_band, n_items = (int64_t)n_q1 * nb2;
  const int64_t n_w = 2 * n_items * n_band;
  CHG_CHECK_ARG(work_doubles >= n_w + (int64_t)CHG_ISE_MAX_CHUNKS * n_t * n_band,
                "work holds less than 2 n_q1 n_band^3 + CHG_ISE_MAX_CHUNKS n_t n_band doubles");
  const int64_t t_tiles = ((int64_t)n_t + ISE_T_TILE - 1) / ISE_T_TILE;
  CHG_CHECK_ARG(n_band <= 65535 && t_tiles <= 65535, "too many bands or temperatures");
  double2* wts = reinterpret_cast<double2*>(work);
  double* partial = work + n_w;
  cudaStream_t st = as_stream(stream);
  ise_weights_kernel<false><<<(unsigned)((n_items + ISE_THREADS - 1) / ISE_THREADS), ISE_THREADS, 0, st>>>(
      freqs, n_band, n1, n2, n3, tetrahedra, target, omega, q1_idx, n_q1, cutoff_thz, wts);
  count_launch();
  // enough chunks for about 4 096 blocks in all, at most CHG_ISE_MAX_CHUNKS and one pass of the block's threads each
  const int64_t others = (int64_t)n_band * t_tiles;
  const int64_t want = (4096 + others - 1) / others;
  const int chunks = (int)std::max<int64_t>(
      1, std::min<int64_t>({(int64_t)CHG_ISE_MAX_CHUNKS, (n_items + ISE_THREADS - 1) / ISE_THREADS, want}));
  ise_accumulate_kernel<<<dim3(chunks, (unsigned)n_band, (unsigned)t_tiles), ISE_THREADS, 0, st>>>(
      freqs, n_band, n1, n2, n3, target, omega, q1_idx, n_q1, p, wts, temperatures, n_t, cutoff_thz, partial);
  CHG_CUDA(reduce_chunks(partial, chunks, (int64_t)n_t * n_band, AccumulateStore{gamma}, st));
  CHG_LAUNCH_END();
}

extern "C" int chg_collision_rows(const double* freqs, int32_t n_band, int32_t n1, int32_t n2, int32_t n3,
                                  const int32_t* tetrahedra, int32_t target, const double* omega, const int32_t* q1_idx,
                                  int32_t n_q1, const double* p, const double* temperatures, int32_t n_t,
                                  double cutoff_thz, double* work, int64_t work_doubles, double* out, void* stream) {
  CHG_CHECK_ARG(n_band >= 0 && n1 > 0 && n2 > 0 && n3 > 0 && n_q1 >= 0 && n_t >= 0, "bad size");
  CHG_CHECK_ARG((int64_t)n1 * n2 * n3 * std::max(n_band, 1) < (1ll << 31), "mesh too large");
  CHG_CHECK_ARG(target >= 0 && (int64_t)target < (int64_t)n1 * n2 * n3, "target outside the mesh");
  CHG_CHECK_ARG(n_band <= COLL_MAX_BAND, "too many bands (at most 768)");
  if (n_band == 0 || n_q1 == 0 || n_t == 0) return CHG_OK;
  CHG_CHECK_ARG(freqs && tetrahedra && omega && q1_idx && p && temperatures && work && out, "null pointer");
  const int64_t n_items = (int64_t)n_q1 * n_band * n_band;
  CHG_CHECK_ARG(work_doubles >= 3 * n_items * n_band, "work holds less than 3 n_q1 n_band^3 doubles");
  const int64_t t_tiles = ((int64_t)n_t + COLL_T_TILE - 1) / COLL_T_TILE;
  CHG_CHECK_ARG(t_tiles <= 65535, "too many temperatures");
  cudaStream_t st = as_stream(stream);
  ise_weights_kernel<true><<<(unsigned)((n_items + ISE_THREADS - 1) / ISE_THREADS), ISE_THREADS, 0, st>>>(
      freqs, n_band, n1, n2, n3, tetrahedra, target, omega, q1_idx, n_q1, cutoff_thz, reinterpret_cast<double2*>(work));
  count_launch();
  const size_t smem = sizeof(double) * 2 * COLL_T_TILE * n_band;
  collision_rows_kernel<<<dim3((unsigned)n_q1, (unsigned)t_tiles), COLL_THREADS, smem, st>>>(
      freqs, n_band, n1, n2, n3, target, q1_idx, n_q1, p, work, temperatures, n_t, cutoff_thz, out);
  CHG_LAUNCH_END();
}

extern "C" int chg_self_energy_spectrum(const double* freqs, int32_t n_band, int32_t n1, int32_t n2, int32_t n3,
                                        const int32_t* tetrahedra, int32_t target, const double* omega, int32_t n_freq,
                                        const int32_t* q1_idx, int32_t n_q1, const double* p,
                                        const double* temperatures, int32_t n_t, double cutoff_thz, double* work,
                                        int64_t work_doubles, double* gamma, void* stream) {
  CHG_CHECK_ARG(n_band >= 0 && n1 > 0 && n2 > 0 && n3 > 0 && n_freq >= 0 && n_q1 >= 0 && n_t >= 0, "bad size");
  CHG_CHECK_ARG((int64_t)n1 * n2 * n3 * std::max(n_band, 1) < (1ll << 31), "mesh too large");
  CHG_CHECK_ARG(target >= 0 && (int64_t)target < (int64_t)n1 * n2 * n3, "target outside the mesh");
  if (n_band == 0 || n_freq == 0 || n_q1 == 0 || n_t == 0) return CHG_OK;
  CHG_CHECK_ARG(freqs && tetrahedra && omega && q1_idx && p && temperatures && work && gamma, "null pointer");
  const int64_t n_out = (int64_t)n_t * n_band * n_freq;
  CHG_CHECK_ARG(work_doubles >= (int64_t)CHG_SE_MAX_CHUNKS * n_out,
                "work holds less than CHG_SE_MAX_CHUNKS n_t n_band n_freq doubles");
  const int64_t f_tiles = ((int64_t)n_freq + SE_F_TILE - 1) / SE_F_TILE;
  const int64_t l_tiles = ((int64_t)n_band + SE_L_TILE - 1) / SE_L_TILE;
  const int64_t t_tiles = ((int64_t)n_t + SE_T_TILE - 1) / SE_T_TILE;
  CHG_CHECK_ARG(f_tiles * l_tiles <= 65535 && t_tiles <= 65535, "too many frequency points, bands or temperatures");
  // enough chunks for about 4 096 blocks in all, at most CHG_SE_MAX_CHUNKS and one item tile each
  const int64_t n_tiles = ((int64_t)n_q1 * n_band * n_band + SE_ITEMS - 1) / SE_ITEMS;
  const int64_t others = f_tiles * l_tiles * t_tiles;
  const int64_t want = (4096 + others - 1) / others;
  const int chunks =
      (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)CHG_SE_MAX_CHUNKS, n_tiles, want}));
  cudaStream_t st = as_stream(stream);
  self_energy_spectrum_kernel<<<dim3(chunks, (unsigned)(f_tiles * l_tiles), (unsigned)t_tiles), SE_THREADS, 0, st>>>(
      freqs, n_band, n1, n2, n3, tetrahedra, target, omega, n_freq, q1_idx, n_q1, p, temperatures, n_t, cutoff_thz,
      work);
  CHG_CUDA(reduce_chunks(work, chunks, n_out, AccumulateStore{gamma}, st));
  CHG_LAUNCH_END();
}

extern "C" int chg_coherence_conductivity(const double* freqs, const double* eigvecs, const double* ddyn,
                                          const int32_t* set_id, const double* heat_capacity, const double* gamma,
                                          int32_t n_q, int32_t n_band, int32_t n_t, double cutoff_thz, double* work,
                                          int64_t work_doubles, double* kappa, void* stream) {
  CHG_CHECK_ARG(n_q >= 0 && n_band >= 0 && n_t >= 0, "negative size");
  if (n_q == 0 || n_band == 0 || n_t == 0) return CHG_OK;
  CHG_CHECK_ARG(freqs && eigvecs && ddyn && set_id && heat_capacity && gamma && work && kappa, "null pointer");
  CHG_CHECK_ARG(n_q <= 65535, "too many q in one call (at most 65535)");
  CHG_CHECK_ARG(n_band <= 46340, "too many bands");
  const int64_t t_tiles = ((int64_t)n_t + COH_T_TILE - 1) / COH_T_TILE;
  CHG_CHECK_ARG(t_tiles <= 65535, "too many temperatures");
  const int64_t nb2 = (int64_t)n_band * n_band, n_v = 3 * (int64_t)n_q * nb2;  // complex elements of W and of V
  CHG_CHECK_ARG(work_doubles >= 4 * n_v + (int64_t)CHG_WIGNER_MAX_CHUNKS * n_t * 6,
                "work holds less than 12 n_q n_band^2 + CHG_WIGNER_MAX_CHUNKS n_t 6 doubles");
  double2* w_buf = reinterpret_cast<double2*>(work);
  double2* v_buf = w_buf + n_v;
  double* partial = work + 4 * n_v;
  const double2* eig = reinterpret_cast<const double2*>(eigvecs);
  // c = THZ_PER_SQRT_EV_A2_AMU of chgnet_b200.phonons: the same expression in the same order
  const double ang = 1e-10;
  const double c = sqrt(1.602176634e-19 / (ang * ang * 1.66053906660e-27)) / (2 * 3.141592653589793) / 1e12;
  const int64_t tiles = ((int64_t)n_band + COH_TILE - 1) / COH_TILE;
  const dim3 ggrid((unsigned)(tiles * tiles), (unsigned)n_q, 3);
  cudaStream_t st = as_stream(stream);
  coh_gemm_kernel<0><<<ggrid, 256, 0, st>>>(eig, reinterpret_cast<const double2*>(ddyn), freqs, n_band, c * c, w_buf);
  count_launch();
  coh_gemm_kernel<1><<<ggrid, 256, 0, st>>>(eig, w_buf, freqs, n_band, c * c, v_buf);
  count_launch();
  const int chunks = std::min(CHG_WIGNER_MAX_CHUNKS, n_q);
  coh_pair_kernel<<<dim3(chunks, (unsigned)t_tiles), COH_THREADS, 0, st>>>(freqs, set_id, v_buf, heat_capacity, gamma,
                                                                          n_q, n_band, n_t, cutoff_thz, partial);
  CHG_CUDA(reduce_chunks(partial, chunks, (int64_t)n_t * 6, SymmetricStore{kappa}, st));
  CHG_LAUNCH_END();
}

extern "C" int chg_isotope_scattering(const double* freqs, const double* eigvecs, int32_t n_band, int32_t n1,
                                      int32_t n2, int32_t n3, const int32_t* tetrahedra, const double* mass_variances,
                                      int32_t n_prim, const int32_t* targets, int32_t n_target, const double* omega,
                                      double cutoff_thz, double* gamma, double* work, int64_t work_doubles,
                                      void* stream) {
  CHG_CHECK_ARG(n_band >= 0 && n1 > 0 && n2 > 0 && n3 > 0 && n_prim >= 0 && n_target >= 0, "bad size");
  CHG_CHECK_ARG(n_band == 3 * n_prim, "n_band must be 3 n_prim");
  const int64_t n_q = (int64_t)n1 * n2 * n3;
  CHG_CHECK_ARG(n_q * 6 * std::max(n_band, 1) < (1ll << 31), "mesh too large");
  CHG_CHECK_ARG(n_target <= 65535, "too many targets in one call (at most 65535)");
  if (n_band == 0 || n_target == 0) return CHG_OK;
  CHG_CHECK_ARG(freqs && eigvecs && tetrahedra && mass_variances && targets && omega && gamma && work, "null pointer");
  const int64_t n_o = (int64_t)n_target * n_q * n_band * n_band;
  CHG_CHECK_ARG(work_doubles >= n_o + (int64_t)CHG_ISO_MAX_CHUNKS * n_target * n_band,
                "work holds less than n_target N n_band^2 + CHG_ISO_MAX_CHUNKS n_target n_band doubles");
  double* partial = work + n_o;
  cudaStream_t st = as_stream(stream);
  iso_overlap_kernel<<<(unsigned)((n_o + ISO_THREADS - 1) / ISO_THREADS), ISO_THREADS, 0, st>>>(
      reinterpret_cast<const double2*>(eigvecs), freqs, n_band, (int)n_q, mass_variances, n_prim, targets, n_target,
      cutoff_thz, work);
  count_launch();
  const int l_tile = std::min(n_band, ISO_THREADS);
  const int l_tiles = (n_band + l_tile - 1) / l_tile;
  // at most CHG_ISO_MAX_CHUNKS chunks of item tiles, at least one tile each: a function of the mesh and n_band only
  const int64_t n_tiles = (n_q * 6 * n_band + ISO_THREADS - 1) / ISO_THREADS;
  const int chunks = (int)std::min<int64_t>(CHG_ISO_MAX_CHUNKS, n_tiles);
  iso_accumulate_kernel<<<dim3(chunks, (unsigned)l_tiles, (unsigned)n_target), ISO_THREADS, 0, st>>>(
      freqs, n_band, n1, n2, n3, tetrahedra, omega, work, n_target, l_tile, cutoff_thz, partial);
  const double scale = 3.141592653589793 / (4.0 * 6.0 * (double)n_q);
  CHG_CUDA(reduce_chunks(partial, chunks, (int64_t)n_target * n_band, IsotopeStore{gamma, omega, scale}, st));
  CHG_LAUNCH_END();
}

extern "C" int chg_sample_displacements(const double* evecs, const double* amp, int32_t n_modes,
                                        const double* inv_sqrt_m, const double* frac_ref, const double* lattice,
                                        const double* inv_lattice, int64_t seed, int64_t iteration,
                                        int64_t first_sample, int32_t n_samples, double* work, int64_t work_doubles,
                                        float* frac, double* u, void* stream) {
  CHG_CHECK_ARG(n_modes >= 0 && n_modes % 3 == 0 && n_samples >= 0, "bad size (n_modes must be 3 n_atoms)");
  CHG_CHECK_ARG(seed >= 0 && iteration >= 0 && first_sample >= 0, "seed, iteration and first_sample must be >= 0");
  if (n_modes == 0 || n_samples == 0) return CHG_OK;
  CHG_CHECK_ARG(evecs && amp && inv_sqrt_m && frac_ref && lattice && inv_lattice && work && frac && u, "null pointer");
  const int64_t tiles_s = ((int64_t)n_samples + EFF_TILE - 1) / EFF_TILE;
  CHG_CHECK_ARG(tiles_s <= 65535, "too many samples in one call (at most 65535 * 64)");
  const int64_t n_xi = (int64_t)n_samples * n_modes;
  CHG_CHECK_ARG(work_doubles >= n_xi, "work holds less than n_samples n_modes doubles");
  cudaStream_t st = as_stream(stream);
  eff_variates_kernel<<<(unsigned)((n_xi + EFF_THREADS - 1) / EFF_THREADS), EFF_THREADS, 0, st>>>(
      amp, n_modes, (uint64_t)seed, (uint64_t)iteration, (uint64_t)first_sample, n_samples, work);
  count_launch();
  const dim3 grid((unsigned)((n_modes + EFF_TILE - 1) / EFF_TILE), (unsigned)tiles_s);
  eff_superpose_kernel<<<grid, EFF_THREADS, 0, st>>>(work, evecs, inv_sqrt_m, n_samples, n_modes, u);
  count_launch();
  const int64_t n_items = (int64_t)n_samples * (n_modes / 3);
  eff_positions_kernel<<<(unsigned)((n_items + EFF_THREADS - 1) / EFF_THREADS), EFF_THREADS, 0, st>>>(
      frac_ref, lattice, inv_lattice, n_modes / 3, n_samples, frac, u);
  CHG_LAUNCH_END();
}

extern "C" int chg_displacement_moments(const double* u, const double* force, const double* f0, const int32_t* perm,
                                        int32_t n_atoms, int32_t n_cells, int32_t n_samples, double* work,
                                        int64_t work_doubles, double* acc, void* stream) {
  CHG_CHECK_ARG(n_atoms >= 0 && n_cells > 0 && n_samples >= 0 && n_atoms % n_cells == 0,
                "bad size (n_atoms must be a multiple of n_cells)");
  CHG_CHECK_ARG(n_samples <= 65535, "too many samples in one call (at most 65535)");
  if (n_atoms == 0 || n_samples == 0) return CHG_OK;
  CHG_CHECK_ARG(u && force && f0 && perm && work && acc, "null pointer");
  const int n_prim = n_atoms / n_cells;
  const int64_t n_out = 18 * (int64_t)n_prim * n_atoms + 2;
  CHG_CHECK_ARG(n_out < (1ll << 31), "supercell too large");
  CHG_CHECK_ARG(work_doubles >= (1 + (int64_t)n_samples) * n_out,
                "work holds less than (1 + n_samples) (18 n_prim n_atoms + 2) doubles");
  cudaStream_t st = as_stream(stream);
  const int64_t pairs = (int64_t)n_prim * n_atoms;
  const dim3 grid((unsigned)((pairs + EFF_THREADS - 1) / EFF_THREADS), (unsigned)n_samples);
  eff_moments_kernel<<<grid, EFF_THREADS, 0, st>>>(u, force, f0, perm, n_atoms, n_cells, n_prim, acc, work);
  CHG_CUDA(reduce_chunks(work, 1 + n_samples, n_out, CopyStore{acc}, st));
  CHG_LAUNCH_END();
}
