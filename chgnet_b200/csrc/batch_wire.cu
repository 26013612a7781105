// Host graphs -> device batch over a COMPACT wire format, packed and shipped in two overlapping phases.
//
// Replaces, for host CrystalGraphs, the concatenation half of BatchedGraph.from_graphs (reference model.py:792-913: one
// `.to(device)` per tensor per graph, index offsets added on the device) and round 1's chg_pack_batch_host + two
// full-size H2D copies.  What crosses PCIe per batch:
//
//   int32  z[N] owner[N] center[Ed] nbr[Ed] d2u[Ed] u2d[Eu] | ang_di[A] ang_dj[A]
//   fp32   frac[3N] lattice[9B]
//   int8   image[3Ed]
//
// i.e. 8 instead of 20 bytes per angle and 3 instead of 12 bytes per neighbour image (c3: 18.7 MB instead of 35.1 MB).
// The three bond-graph columns that are functions of the two directed-edge columns,
//     ang_atom = center[ang_di],  ang_i = d2u[ang_di],  ang_j = d2u[ang_dj]          (graph.py:233-277 builds them so),
// and the fp32 images are re-created on the device by two tiny kernels.  The packer VERIFIES both assumptions for every
// angle / image while it reads them (flags_out[4] != 0: some graph does not satisfy them -> nothing usable was
// produced and the caller falls back to chg_pack_batch_host, which ships every column as given).
//
// Phase 1 packs atoms, edges and bonds; its three copies are enqueued and run while phase 2 packs the angles.  Worker
// threads are persistent (parked on a condition variable between batches).
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#include <unistd.h>

#include "common.cuh"
#include "worker_pool.h"

#define CHG_LAUNCH_CHECK(what)                                                      \
  do {                                                                              \
    cudaError_t _e = cudaGetLastError();                                            \
    if (_e != cudaSuccess) {                                                        \
      chg::set_error("%s: launch failed: %s", what, cudaGetErrorString(_e));        \
      return CHG_ERR_CUDA;                                                          \
    }                                                                               \
    chg::count_launch();                                                            \
  } while (0)

namespace chg {
namespace {

// ---- device side: re-create what was not shipped -------------------------------------------------------------------
__global__ void expand_image_kernel(const int8_t* __restrict__ img8, float* __restrict__ image, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    image[i] = (float)img8[i];
}

__global__ void derive_angle_columns_kernel(const int32_t* __restrict__ center, const int32_t* __restrict__ d2u,
                                            const int32_t* __restrict__ ang_di, const int32_t* __restrict__ ang_dj,
                                            int32_t* __restrict__ ang_atom, int32_t* __restrict__ ang_i,
                                            int32_t* __restrict__ ang_j, int32_t n) {
  for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < n; a += gridDim.x * blockDim.x) {
    const int di = ang_di[a], dj = ang_dj[a];
    ang_atom[a] = __ldg(center + di);
    ang_i[a] = __ldg(d2u + di);
    ang_j[a] = __ldg(d2u + dj);
  }
}

}  // namespace
}  // namespace chg

using namespace chg;

// Pinned staging memory for the packers.  write_combined != 0: cudaHostAllocWriteCombined - the packer's worker threads
// only WRITE it (streaming stores, no cache lines left dirty in many cores' caches), and the copy engine reads it at
// full PCIe rate (on the earlier Blackwell build's hosts a 19 MiB buffer freshly written by 8 threads copied at 54 GB/s
// from write-combined memory and at 8 GB/s from ordinary pinned memory).  Never read it on the CPU.
extern "C" int chg_host_alloc(int64_t bytes, int32_t write_combined, void** out) {
  CHG_CHECK_ARG(bytes > 0 && out != nullptr, "bad size or null pointer");
  CHG_CUDA(cudaHostAlloc(out, (size_t)bytes, write_combined ? cudaHostAllocWriteCombined : cudaHostAllocDefault));
  return CHG_OK;
}

extern "C" int chg_host_free(void* p) {
  if (p != nullptr) CHG_CUDA(cudaFreeHost(p));
  return CHG_OK;
}

// counts [B][4] = atoms, directed edges, bonds, angles per graph; ptrs [B][8] = z (int32), frac (fp32 [n][3]),
// atom_graph (int32 [ed][2]), image (fp32 [ed][3]), d2u, u2d (int32), bond_graph (int32 [an][5]), lattice (fp32 [9]).
// Host staging (pinned): ibuf_host [2N + 3Ed + Eu + 2A], fbuf_host [3N + 9B], img_host [3Ed].
// Device (or all three NULL: pack only, for tests without a GPU): ibuf_dev [2N + 3Ed + Eu + 5A] = the host layout followed
// by ang_atom[A] ang_i[A] ang_j[A]; fbuf_dev [3N + 9B + 3Ed] = frac, lattice, image; img_dev [3Ed].
// flags_out[0..3] as chg_pack_batch_host; flags_out[4] = 0, or the reason the compact format does not apply
// (1 image not a small integer, 2 bond-graph columns not derivable, 3 bond-graph edge index out of range).
extern "C" int chg_pack_batch_wire(int32_t n_graphs, const int64_t* counts, const void* const* ptrs, int32_t* ibuf_host,
                                   float* fbuf_host, int8_t* img_host, int32_t* ibuf_dev, float* fbuf_dev, int8_t* img_dev,
                                   int32_t* flags_out, void* stream_) {
  CHG_CHECK_ARG(n_graphs >= 0, "negative size");
  CHG_CHECK_ARG(counts != nullptr && ptrs != nullptr && ibuf_host != nullptr && fbuf_host != nullptr && img_host != nullptr &&
                    flags_out != nullptr,
                "null pointer");
  const bool ship = ibuf_dev != nullptr;
  CHG_CHECK_ARG(!ship || (fbuf_dev != nullptr && img_dev != nullptr), "null device pointer");
  cudaStream_t stream = as_stream(stream_);

  std::vector<int64_t> off((size_t)(n_graphs + 1) * 4, 0);
  for (int g = 0; g < n_graphs; ++g)
    for (int k = 0; k < 4; ++k) off[(size_t)(g + 1) * 4 + k] = off[(size_t)g * 4 + k] + counts[4 * g + k];
  const int64_t N = off[(size_t)n_graphs * 4], Ed = off[(size_t)n_graphs * 4 + 1], Eu = off[(size_t)n_graphs * 4 + 2],
                A = off[(size_t)n_graphs * 4 + 3];
  CHG_CHECK_ARG(N < INT32_MAX && Ed < INT32_MAX / 3 && A < INT32_MAX, "batch too large for int32 indices");
  int32_t* z = ibuf_host;
  int32_t* owner = z + N;
  int32_t* center = owner + N;
  int32_t* nbr = center + Ed;
  int32_t* d2u = nbr + Ed;
  int32_t* u2d = d2u + Ed;
  int32_t* ang_di = u2d + Eu;
  int32_t* ang_dj = ang_di + A;
  float* frac = fbuf_host;
  float* lattice = frac + N * 3;
  const int64_t n_int_1 = 2 * N + 3 * Ed + Eu, n_flt = 3 * N + 9 * (int64_t)n_graphs;
  static thread_local std::vector<uint8_t> in_bond_graph;
  in_bond_graph.assign((size_t)Eu, 0);
  uint8_t* bg_flag = in_bond_graph.data();

  struct Partial {
    bool edges_sorted = true, angles_sorted = true;
    int64_t bad_z = -1, n_short = 0;
    int reject = 0;
  };
  const int64_t total_items = N * 5 + Ed * 6 + Eu + A * 5;
  WorkerPool& wp = pool();
  int n_thr = 1;
  if (total_items > (1 << 18)) n_thr = (int)std::min<int64_t>(wp.size(), std::max<int64_t>(1, total_items >> 17));
  // work units: 4 per worker, taken from a shared counter, so that a worker the host deschedules for a while (busy box)
  // delays one small unit, not a sixteenth of the batch.  Many graphs: unit t = the graphs cut[t] .. cut[t+1]-1, whole;
  // few (large) graphs: unit t = slice t of every array of every graph.
  const bool by_graph = n_graphs >= 4 * n_thr;
  const int n_units = n_thr == 1 ? 1 : (by_graph ? (int)std::min<int64_t>(n_graphs, 4 * n_thr) : 4 * n_thr);
  std::vector<int> cut((size_t)n_units + 1, n_graphs);
  cut[0] = 0;
  if (by_graph) {
    auto weight = [&](int g) { return off[(size_t)g * 4] * 5 + off[(size_t)g * 4 + 1] * 6 + off[(size_t)g * 4 + 2] + off[(size_t)g * 4 + 3] * 5; };
    for (int t = 1, g = 0; t < n_units; ++t) {
      const int64_t target = total_items * t / n_units;
      while (g < n_graphs && weight(g) < target) ++g;
      cut[t] = g;
    }
  }
  std::vector<Partial> parts((size_t)n_units);

  auto phase = [&](int which, int t) {
    Partial& res = parts[t];
    const int g0 = by_graph ? cut[t] : 0, g1 = by_graph ? cut[t + 1] : n_graphs;
    const int part = by_graph ? 0 : t, nparts = by_graph ? 1 : n_units;
    for (int g = g0; g < g1; ++g) {
      const int64_t n = counts[4 * g], ed = counts[4 * g + 1], eu = counts[4 * g + 2], an = counts[4 * g + 3];
      const int64_t a_off = off[(size_t)g * 4], e_off = off[(size_t)g * 4 + 1], u_off = off[(size_t)g * 4 + 2], g_off = off[(size_t)g * 4 + 3];
      const void* const* p = ptrs + 8 * g;
      auto lo = [&](int64_t len) { return len * part / nparts; };
      auto hi = [&](int64_t len) { return len * (part + 1) / nparts; };
      const int32_t* ag = static_cast<const int32_t*>(p[2]);
      const int32_t* du = static_cast<const int32_t*>(p[4]);
      if (which == 0) {
        if (n > 0) {
          const int64_t i0 = lo(n), i1 = hi(n);
          const int32_t* zs = static_cast<const int32_t*>(p[0]);
          std::memcpy(z + a_off + i0, zs + i0, (size_t)(i1 - i0) * 4);
          std::memcpy(frac + (a_off + i0) * 3, static_cast<const float*>(p[1]) + i0 * 3, (size_t)(i1 - i0) * 12);
          for (int64_t i = i0; i < i1; ++i) {
            owner[a_off + i] = g;
            if ((zs[i] < 1 || zs[i] > CHG_MAX_Z) && res.bad_z < 0) res.bad_z = a_off + i;
          }
        }
        // one output array per loop: the staging buffer may be write-combined memory, which only combines stores into full
        // lines while a core writes ONE stream at a time (the sources stay in L1 / L2 between the loops)
        const float* im = static_cast<const float*>(p[3]);
        const int64_t e0 = lo(ed), e1 = hi(ed);
        for (int64_t e = e0; e < e1; ++e) {
          center[e_off + e] = ag[2 * e] + (int32_t)a_off;
          if (e > 0 && ag[2 * e] < ag[2 * e - 2]) res.edges_sorted = false;
        }
        for (int64_t e = e0; e < e1; ++e) nbr[e_off + e] = ag[2 * e + 1] + (int32_t)a_off;
        for (int64_t e = e0; e < e1; ++e) d2u[e_off + e] = du[e] + (int32_t)u_off;
        for (int64_t i = 3 * e0; i < 3 * e1; ++i) {
          const float v = im[i];
          const int8_t q = (v >= -127.f && v <= 127.f) ? (int8_t)v : (int8_t)0;
          if ((float)q != v) res.reject = 1;
          img_host[e_off * 3 + i] = q;
        }
        const int32_t* ud = static_cast<const int32_t*>(p[5]);
        for (int64_t u = lo(eu); u < hi(eu); ++u) u2d[u_off + u] = ud[u] + (int32_t)e_off;
        if (part == 0) std::memcpy(lattice + (size_t)g * 9, p[7], 36);
      } else {
        const int32_t* bg = static_cast<const int32_t*>(p[6]);
        const int64_t a0 = lo(an), a1 = hi(an);
        for (int64_t a = a0; a < a1; ++a) {
          const int64_t di = bg[5 * a + 2], dj = bg[5 * a + 4];
          if (di < 0 || di >= ed || dj < 0 || dj >= ed) {
            res.reject = 3;
            ang_di[g_off + a] = 0;
            continue;
          }
          if (bg[5 * a] != ag[2 * di] || bg[5 * a + 1] != du[di] || bg[5 * a + 3] != du[dj]) res.reject = 2;
          ang_di[g_off + a] = (int32_t)(di + e_off);
          if (a > 0 && bg[5 * a + 1] < bg[5 * a - 4]) res.angles_sorted = false;
          for (int which_bond = 1; which_bond <= 3; which_bond += 2) {
            const int64_t ul = bg[5 * a + which_bond];
            if (ul >= 0 && ul < eu && __atomic_exchange_n(&bg_flag[u_off + ul], (uint8_t)1, __ATOMIC_RELAXED) == 0) ++res.n_short;
          }
        }
        for (int64_t a = a0; a < a1; ++a) ang_dj[g_off + a] = bg[5 * a + 4] + (int32_t)e_off;
      }
    }
  };

  auto reduce_flags = [&]() {
    bool edges_sorted = true, angles_sorted = true;
    int64_t bad_z = -1, n_short = 0;
    int reject = 0;
    for (const Partial& r : parts) {
      edges_sorted = edges_sorted && r.edges_sorted;
      angles_sorted = angles_sorted && r.angles_sorted;
      if (r.bad_z >= 0 && (bad_z < 0 || r.bad_z < bad_z)) bad_z = r.bad_z;
      n_short += r.n_short;
      if (r.reject != 0 && reject == 0) reject = r.reject;
    }
    flags_out[0] = edges_sorted ? 1 : 0;
    flags_out[1] = angles_sorted ? 1 : 0;
    flags_out[2] = (int32_t)bad_z;
    flags_out[3] = (int32_t)n_short;
    flags_out[4] = reject;
    return reject;
  };

  // ---- phase 1: atoms, edges, bonds -> three copies in flight while the angles are packed -------------------------
  auto run_phase = [&](int which) {
    std::atomic<int> next{0};
    wp.run(n_thr, [&](int) {
      for (int u = next.fetch_add(1, std::memory_order_relaxed); u < n_units; u = next.fetch_add(1, std::memory_order_relaxed)) phase(which, u);
    });
  };
  run_phase(0);
  if (reduce_flags() != 0 || flags_out[2] >= 0) return CHG_OK;  // compact format rejected / bad Z: nothing shipped
  if (ship) {
    if (n_int_1 > 0) CHG_CUDA(cudaMemcpyAsync(ibuf_dev, ibuf_host, (size_t)n_int_1 * 4, cudaMemcpyHostToDevice, stream));
    if (n_flt > 0) CHG_CUDA(cudaMemcpyAsync(fbuf_dev, fbuf_host, (size_t)n_flt * 4, cudaMemcpyHostToDevice, stream));
    if (Ed > 0) {
      CHG_CUDA(cudaMemcpyAsync(img_dev, img_host, (size_t)Ed * 3, cudaMemcpyHostToDevice, stream));
      const int64_t n_img = Ed * 3;
      expand_image_kernel<<<(unsigned)std::min<int64_t>((n_img + 255) / 256, 4 * sm_count()), 256, 0, stream>>>(img_dev, fbuf_dev + n_flt, n_img);
      CHG_LAUNCH_CHECK("chg_pack_batch_wire (expand_image)");
    }
  }
  // ---- phase 2: angles ---------------------------------------------------------------------------------------------
  if (A > 0) run_phase(1);
  if (reduce_flags() != 0) {
    if (ship) cudaStreamSynchronize(stream);  // the caller re-packs into the same staging buffers
    return CHG_OK;
  }
  if (ship && A > 0) {
    CHG_CUDA(cudaMemcpyAsync(ibuf_dev + n_int_1, ibuf_host + n_int_1, (size_t)A * 8, cudaMemcpyHostToDevice, stream));
    int32_t* dev_center = ibuf_dev + 2 * N;
    int32_t* dev_d2u = dev_center + 2 * Ed;
    int32_t* dev_di = ibuf_dev + n_int_1;
    derive_angle_columns_kernel<<<(unsigned)std::min<int64_t>((A + 255) / 256, 4 * sm_count()), 256, 0, stream>>>(
        dev_center, dev_d2u, dev_di, dev_di + A, dev_di + 2 * A, dev_di + 3 * A, dev_di + 4 * A, (int32_t)A);
    CHG_LAUNCH_CHECK("chg_pack_batch_wire (derive_angle_columns)");
  }
  return CHG_OK;
}
