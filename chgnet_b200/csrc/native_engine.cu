// Whole-path entry points of the C ABI: weight packing and ONE call for forward (+ force / stress).
//
// `chg_forward` runs the kernel schedule of chgnet_b200/engine.py (Engine.run, inference) natively:
// the same per-kernel entry points, in the same order, on a caller-provided workspace — what a
// non-Python host (or the reference's own model.py through one ctypes call) would bind instead of
// `CHGNet._compute` + the two `torch.autograd.grad` calls (reference model.py:389-542).
// `chg_pack_weights_host` is weights.py::pack_weights for a host-side state_dict.
//
// Memory: nothing is allocated.  `chg_forward_plan` replays the schedule without launching anything
// and returns the workspace size (and, for tests, the list of calls); `chg_forward` bump-allocates
// from the workspace: saved-for-reverse buffers from the bottom, per-layer temporaries from the top.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>

#include "common.cuh"

namespace chg {
namespace {

constexpr size_t ALIGN = 256;  // bytes
constexpr int64_t PAD = 16;    // floats: every packed piece starts on a 64-byte boundary

struct GatedW {
  const float *w2t = nullptr, *w2 = nullptr, *b2 = nullptr, *ln = nullptr;
  const float *a_t = nullptr, *b_t = nullptr, *c_t = nullptr, *bias1 = nullptr;  // first layer, k-major blocks
  const float *a_b = nullptr, *b_b = nullptr, *c_b = nullptr;                    // same, PyTorch layout (reverse)
  const float *wo_t = nullptr, *wo = nullptr, *bo = nullptr;
};
struct Weights {
  const float *emb, *freq_ag, *freq_bg, *freq_ang, *w3t, *w3, *wang_t, *wang;
  GatedW atom[CHG_MAX_CONV], bond[CHG_MAX_CONV], angle[CHG_MAX_CONV];
  const float *readout_ln, *mlp_wt, *mlp_w, *mlp_b, *w_last, *w_mag, *atom_ref;
};

// One walk defines the blob layout for the host packer and the device view alike.
struct Walker {
  float* base;
  int64_t off = 0;
  float* take(int64_t n) {
    float* p = base == nullptr ? nullptr : base + off;
    off += (n + PAD - 1) / PAD * PAD;
    return p;
  }
};

int64_t walk(const chg_hparams& hp, float* base, Weights& w) {
  Walker k{base};
  const int R = hp.num_radial, NA = hp.num_angular, F = (NA - 1) / 2, L = hp.n_readout_hidden;
  w.emb = k.take(94 * 64);
  w.freq_ag = k.take(R);
  w.freq_bg = k.take(R);
  w.freq_ang = k.take(F);
  w.w3t = k.take(3 * R * 64);
  w.w3 = k.take(3 * 64 * R);
  w.wang_t = k.take(NA * 64);
  w.wang = k.take(64 * NA);
  auto second = [&](GatedW& g) {
    g.w2t = k.take(64 * 128);
    g.w2 = k.take(128 * 64);
    g.b2 = k.take(128);
  };
  for (int t = 0; t < hp.n_conv; ++t) {
    GatedW& g = w.atom[t];
    second(g);
    g.ln = hp.use_ln ? k.take(256) : nullptr;
    g.a_t = k.take(64 * 256);  // wcn_t
    g.b_t = k.take(64 * 128);  // we_t
    g.bias1 = k.take(128);
    g.a_b = k.take(256 * 64);
    g.b_b = k.take(128 * 64);
    g.wo_t = k.take(4096);
    g.wo = k.take(4096);
    g.bo = hp.has_mlp_out_bias ? k.take(64) : nullptr;
  }
  for (int t = 0; t < hp.n_conv - 1; ++t) {
    for (int kind = 0; kind < 2; ++kind) {
      GatedW& g = kind == 0 ? w.bond[t] : w.angle[t];
      if (kind == 0) second(g);
      g.ln = hp.use_ln ? k.take(256) : nullptr;
      g.a_t = k.take(64 * 256);  // wij_t
      g.bias1 = k.take(256);     // bij (bias rides on the i half)
      g.b_t = k.take(64 * 128);  // wx_t
      g.c_t = k.take(64 * 128);  // w1a_t
      g.a_b = k.take(256 * 64);
      g.b_b = k.take(128 * 64);
      g.c_b = k.take(128 * 64);
      if (kind == 0) {
        g.wo_t = k.take(4096);
        g.wo = k.take(4096);
        g.bo = hp.has_mlp_out_bias ? k.take(64) : nullptr;
      }
    }
  }
  w.readout_ln = hp.readout_ln ? k.take(128) : nullptr;
  w.mlp_wt = k.take((int64_t)L * 4096);
  w.mlp_w = k.take((int64_t)L * 4096);
  w.mlp_b = k.take((int64_t)L * 64);
  w.w_last = k.take(64);
  w.w_mag = k.take(64);
  w.atom_ref = k.take(94);
  return k.off;
}

bool hp_ok(const chg_hparams* hp) {
  return hp != nullptr && hp->num_radial >= 1 && hp->num_radial <= 32 && hp->num_angular >= 1 && hp->num_angular <= 31 &&
         (hp->num_angular & 1) && hp->n_conv >= 1 && hp->n_conv <= CHG_MAX_CONV && hp->n_readout_hidden >= 1 &&
         hp->n_readout_hidden <= 4;
}

// ---- host packing helpers (weights.py: _cat_t and torch.cat(dim=0)) ---------------------------------
inline float* mut(const float* p) { return const_cast<float*>(p); }
// dst [64][ld] (k-major), columns col..col+63  <-  W[o][c0 + k]   (W is [64][ldw])
void put_t(const float* dst_c, int ld, int col, const float* W, int ldw, int c0) {
  float* dst = mut(dst_c);
  for (int o = 0; o < 64; ++o)
    for (int kk = 0; kk < 64; ++kk) dst[(size_t)kk * ld + col + o] = W[(size_t)o * ldw + c0 + kk];
}
// dst rows blk*64 .. +63 of a [.][64] matrix  <-  W[o][c0 + k]
void put_rows(const float* dst_c, int blk, const float* W, int ldw, int c0) {
  float* dst = mut(dst_c);
  for (int o = 0; o < 64; ++o)
    for (int kk = 0; kk < 64; ++kk) dst[((size_t)blk * 64 + o) * 64 + kk] = W[(size_t)o * ldw + c0 + kk];
}
void copy_n(const float* dst, const float* src, int n) { std::memcpy(mut(dst), src, sizeof(float) * n); }

void pack_second(const GatedW& g, const chg_gated_sd& s) {
  put_t(g.w2t, 128, 0, s.core_w2, 64, 0);
  put_t(g.w2t, 128, 64, s.gate_w2, 64, 0);
  put_rows(g.w2, 0, s.core_w2, 64, 0);
  put_rows(g.w2, 1, s.gate_w2, 64, 0);
  copy_n(g.b2, s.core_b2, 64);
  copy_n(g.b2 + 64, s.gate_b2, 64);
}
void pack_ln(const GatedW& g, const chg_gated_sd& s) {
  if (g.ln == nullptr) return;
  copy_n(g.ln, s.ln1_w, 64);
  copy_n(g.ln + 64, s.ln1_b, 64);
  copy_n(g.ln + 128, s.ln2_w, 64);
  copy_n(g.ln + 192, s.ln2_b, 64);
}
void pack_out(const GatedW& g, const chg_gated_sd& s) {
  put_t(g.wo_t, 64, 0, s.out_w, 64, 0);
  copy_n(g.wo, s.out_w, 4096);
  if (g.bo != nullptr) copy_n(g.bo, s.out_b, 64);
}

// ---- workspace ---------------------------------------------------------------------------------------
struct Arena {
  char* base = nullptr;
  size_t cap = 0, lo = 0, top_used = 0, peak = 0;
  bool dry = false, overflow = false;
  static size_t up(size_t b) { return (b + ALIGN - 1) / ALIGN * ALIGN; }
  void note() {
    if (lo + top_used > peak) peak = lo + top_used;
    if (!dry && lo + top_used > cap) overflow = true;
  }
  void* keep(size_t bytes) {  // lives until the end of the call
    void* p = dry ? nullptr : base + lo;
    lo += up(bytes);
    note();
    return p;
  }
  void* tmp(size_t bytes) {  // lives until the next reset_tmp()
    top_used += up(bytes);
    note();
    return (dry || overflow) ? nullptr : base + (cap - top_used);
  }
  void reset_tmp() { top_used = 0; }
};

struct Ctx {
  Arena ar;
  cudaStream_t stream = nullptr;
  std::string* trace = nullptr;
  int rc = CHG_OK;
  float* f(bool keep, size_t n) { return static_cast<float*>(keep ? ar.keep(n * 4) : ar.tmp(n * 4)); }
  bool go(const char* name) {  // true -> launch
    if (trace != nullptr) {
      trace->append(name);
      trace->push_back('\n');
    }
    return !ar.dry && !ar.overflow && rc == CHG_OK;
  }
  void zero(void* p, size_t bytes) {
    if (!ar.dry && !ar.overflow && rc == CHG_OK && bytes > 0 && cudaMemsetAsync(p, 0, bytes, stream) != cudaSuccess) {
      set_error("chg_forward: cudaMemsetAsync failed");
      rc = CHG_ERR_CUDA;
    }
  }
};

#define RUN(c, name, call) \
  do {                     \
    if ((c).go(name)) (c).rc = (call); \
  } while (0)

int run_schedule(const chg_hparams& hp, const Weights& W, const chg_batch& b, const chg_outputs& o, Ctx& c) {
  const int N = b.n_atoms, Ed = b.n_edges, Eu = b.n_bonds, A = b.n_angles, B = b.n_graphs, Es = b.n_short;
  const bool has_ang = A > 0;
  const bool grad = o.force != nullptr || o.virial != nullptr;
  const int n_conv = hp.n_conv;
  void* st = c.stream;
  auto lin = [&](const float* x, const int32_t* xr, int m, int k, const float* wt, const float* bias, const float* res,
                 const int32_t* yr, int n, float* y) { RUN(c, "linear", chg_linear(x, xr, m, k, wt, bias, res, yr, n, y, st)); };
  auto seg = [&](const float* data, int width, const int32_t* perm, const int32_t* ptr, int rows, int items, int acc,
                 float* out, int ld) { RUN(c, "segment_sum", chg_segment_sum(data, width, perm, ptr, rows, items, acc, out, ld, st)); };

  // ---- geometry, bases, embeddings
  float* x = c.f(true, (size_t)N * 64);
  RUN(c, "embed_atoms", chg_embed_atoms(b.z, W.emb, N, x, st));
  float *rvec = c.f(true, (size_t)Ed * 3), *dist = c.f(true, Ed), *rhat = c.f(true, (size_t)Ed * 3);
  RUN(c, "edge_geometry", chg_edge_geometry(b.frac, b.lattice, b.owner, b.center, b.nbr, b.image, Ed, rvec, dist, rhat, st));
  float *e = c.f(true, (size_t)Eu * 64), *wag = c.f(true, (size_t)Eu * 64), *wbg = c.f(true, (size_t)Eu * 64);
  RUN(c, "bond_basis_embed", chg_bond_basis_embed(dist, b.u2d, Eu, W.freq_ag, W.freq_bg, hp.num_radial, hp.atom_graph_cutoff,
                                                  hp.bond_graph_cutoff, hp.cutoff_coeff, W.w3t, e, wag, wbg, nullptr, st));
  float *ang = nullptr, *ang_alt = nullptr, *wbg_s = nullptr;
  if (has_ang) {
    ang = c.f(true, (size_t)A * 64);
    ang_alt = c.f(true, (size_t)A * 64);
    RUN(c, "angle_basis_embed", chg_angle_basis_embed(rhat, b.ang_di, b.ang_dj, A, W.freq_ang, (hp.num_angular - 1) / 2,
                                                      W.wang_t, ang, nullptr, st));
    wbg_s = c.f(true, (size_t)Es * 64);
    RUN(c, "gather_rows", chg_gather_rows(wbg, b.short_ids, Es, 64, wbg_s, st));
  }
  struct SavedAtom { float *pcn, *pe, *p; } sa[CHG_MAX_CONV];
  struct SavedBond { float *pre, *p; } sb[CHG_MAX_CONV];
  float* sang[CHG_MAX_CONV];

  auto atom_conv = [&](int t, const float* xin, float* xout) {
    const GatedW& g = W.atom[t];
    float* pcn = c.f(grad, (size_t)N * 256);
    float* pe = c.f(grad, (size_t)Eu * 128);
    lin(xin, nullptr, N, 64, g.a_t, nullptr, nullptr, nullptr, 256, pcn);
    lin(e, nullptr, Eu, 64, g.b_t, g.bias1, nullptr, nullptr, 128, pe);
    float* save_p = grad ? c.f(true, (size_t)Ed * 128) : nullptr;
    float* agg = c.f(false, (size_t)N * 64);
    float* work = c.f(false, (size_t)chg_gated_fused_workspace_floats(Ed));
    // message + aggregation in one kernel (gated_ws.cu): the [Ed][64] message never reaches HBM
    RUN(c, "atom_conv_fused", chg_atom_conv_fused(pcn, pe, wag, b.center, b.nbr, b.d2u, b.ptr_c, Ed, N, g.w2t, g.b2, g.ln, agg, save_p,
                                                  work, st));
    sa[t] = SavedAtom{pcn, pe, save_p};
    lin(agg, nullptr, N, 64, g.wo_t, g.bo, xin, nullptr, 64, xout);
    c.ar.reset_tmp();
  };

  float* x_mag = nullptr;
  for (int t = 0; t < n_conv - 1; ++t) {
    float* xn = (t == n_conv - 2 && o.atom_fea != nullptr) ? o.atom_fea : c.f(true, (size_t)N * 64);
    atom_conv(t, x, xn);
    x = xn;
    if (has_ang) {
      const GatedW& g = W.bond[t];
      float* pij = c.f(false, (size_t)Es * 256);
      float* px = c.f(false, (size_t)N * 128);
      float* pa = c.f(false, (size_t)A * 128);
      lin(e, b.short_ids, Es, 64, g.a_t, g.bias1, nullptr, nullptr, 256, pij);
      lin(x, nullptr, N, 64, g.b_t, nullptr, nullptr, nullptr, 128, px);
      lin(ang, nullptr, A, 64, g.c_t, nullptr, nullptr, nullptr, 128, pa);
      float* s_pre = grad ? c.f(true, (size_t)A * 128) : nullptr;
      float* s_p = grad ? c.f(true, (size_t)A * 128) : nullptr;
      float* agg = c.f(false, (size_t)Es * 64);
      float* work = c.f(false, (size_t)chg_gated_fused_workspace_floats(A));
      RUN(c, "bond_conv_fused", chg_bond_conv_fused(pij, px, pa, wbg_s, b.ang_atom, b.ang_is, b.ang_js, b.ptr_is, A, Es, g.w2t, g.b2,
                                                    g.ln, agg, s_pre, s_p, work, st));
      lin(agg, nullptr, Es, 64, g.wo_t, g.bo, e, b.short_ids, 64, e);  // e[sid] += Wo agg (+ bias)
      sb[t] = SavedBond{s_pre, s_p};
      c.ar.reset_tmp();
      if (t < n_conv - 2) {  // the last AngleUpdate is dead compute (model.py:470-496)
        const GatedW& ga = W.angle[t];
        pij = c.f(false, (size_t)Es * 256);
        px = c.f(false, (size_t)N * 128);
        pa = c.f(false, (size_t)A * 128);
        lin(e, b.short_ids, Es, 64, ga.a_t, ga.bias1, nullptr, nullptr, 256, pij);
        lin(x, nullptr, N, 64, ga.b_t, nullptr, nullptr, nullptr, 128, px);
        lin(ang, nullptr, A, 64, ga.c_t, nullptr, nullptr, nullptr, 128, pa);
        float* s_pa = grad ? c.f(true, (size_t)A * 128) : nullptr;
        RUN(c, "angle_update_fwd", chg_angle_update_fwd(pij, px, pa, ang, b.ang_atom, b.ang_is, b.ang_js, A, ga.ln, ang_alt, s_pa, st));
        sang[t] = s_pa;
        float* sw = ang;
        ang = ang_alt;
        ang_alt = sw;
        c.ar.reset_tmp();
      }
    }
    if (t == n_conv - 2) {
      x_mag = x;
      if (o.magmom != nullptr) RUN(c, "magmom", chg_magmom(x, N, W.w_mag, hp.b_mag, o.magmom, st));
    }
  }
  if (n_conv == 1 && o.magmom != nullptr) c.zero(o.magmom, (size_t)N * 4);
  (void)x_mag;
  {
    float* xn = c.f(true, (size_t)N * 64);
    atom_conv(n_conv - 1, x, xn);
    x = xn;
  }

  // ---- readout
  float* h_out = o.crystal_fea != nullptr ? c.f(false, (size_t)N * 64) : nullptr;
  float* g_x = grad ? c.f(true, (size_t)N * 64) : nullptr;
  c.zero(o.energy, (size_t)B * 8);
  c.zero(o.e_ref, (size_t)B * 8);
  RUN(c, "readout", chg_readout(x, b.z, b.owner, N, W.readout_ln, W.mlp_wt, W.mlp_w, W.mlp_b, hp.n_readout_hidden, W.w_last,
                                hp.b_last, W.atom_ref, o.site_e, h_out, o.energy, o.e_ref, g_x, st));
  if (o.crystal_fea != nullptr) seg(h_out, 64, nullptr, b.graph_ptr, B, N, 0, o.crystal_fea, 64);
  c.ar.reset_tmp();
  if (!grad) return c.rc;

  // ======================= reverse pass: dE/dr per directed edge -> force, virial =======================
  float* g_e = c.f(true, (size_t)Eu * 64);
  bool g_e_live = false;
  float* g_wag = c.f(true, (size_t)Eu * 64);
  c.zero(g_wag, (size_t)Eu * 256);
  float* g_wbg = has_ang ? c.f(true, (size_t)Es * 64) : nullptr;
  if (has_ang) c.zero(g_wbg, (size_t)Es * 256);
  float* g_a = has_ang ? c.f(true, (size_t)A * 64) : nullptr;
  bool g_a_live = false;

  auto atom_bwd = [&](int t) {
    const GatedW& g = W.atom[t];
    float* g_agg = c.f(false, (size_t)N * 64);
    lin(g_x, nullptr, N, 64, g.wo, nullptr, nullptr, nullptr, 64, g_agg);
    float* g_pre = c.f(false, (size_t)Ed * 128);
    float* g_w = c.f(false, (size_t)Ed * 64);
    RUN(c, "atom_conv_bwd", chg_atom_conv_bwd(sa[t].pcn, sa[t].pe, wag, b.center, b.nbr, b.d2u, Ed, sa[t].p, g_agg, g.w2, g.ln,
                                              g_pre, g_w, nullptr, nullptr, st));
    float* sp = c.f(false, (size_t)N * 256);
    seg(g_pre, 128, nullptr, b.ptr_c, N, Ed, 0, sp, 256);
    seg(g_pre, 128, b.perm_n, b.ptr_n, N, Ed, 0, sp + 128, 256);
    lin(sp, nullptr, N, 256, g.a_b, nullptr, g_x, nullptr, 64, g_x);  // g_x += sp @ Wcn
    float* spe = c.f(false, (size_t)Eu * 128);
    seg(g_pre, 128, b.perm_u, b.ptr_u, Eu, Ed, 0, spe, 128);
    lin(spe, nullptr, Eu, 128, g.b_b, nullptr, g_e_live ? g_e : nullptr, nullptr, 64, g_e);
    g_e_live = true;
    seg(g_w, 64, b.perm_u, b.ptr_u, Eu, Ed, 1, g_wag, 64);
    c.ar.reset_tmp();
  };
  auto angle_scatter = [&](const float* g_pre, const GatedW& g) {
    float* sp = c.f(false, (size_t)Es * 256);
    seg(g_pre, 128, nullptr, b.ptr_is, Es, A, 0, sp, 256);
    seg(g_pre, 128, b.perm_js, b.ptr_js, Es, A, 0, sp + 128, 256);
    lin(sp, nullptr, Es, 256, g.a_b, nullptr, g_e, b.short_ids, 64, g_e);  // g_e[sid] += sp @ Wij
    float* spx = c.f(false, (size_t)N * 128);
    seg(g_pre, 128, b.perm_x, b.ptr_x, N, A, 0, spx, 128);
    lin(spx, nullptr, N, 128, g.b_b, nullptr, g_x, nullptr, 64, g_x);
  };

  atom_bwd(n_conv - 1);
  for (int t = n_conv - 2; t >= 0; --t) {
    if (has_ang) {
      if (t < n_conv - 2) {
        const GatedW& ga = W.angle[t];
        float* g_pre = c.f(false, (size_t)A * 128);
        RUN(c, "angle_update_bwd", chg_angle_update_bwd(sang[t], g_a_live ? g_a : nullptr, A, ga.ln, g_pre, nullptr, st));
        lin(g_pre, nullptr, A, 128, ga.c_b, nullptr, g_a_live ? g_a : nullptr, nullptr, 64, g_a);
        g_a_live = true;
        angle_scatter(g_pre, ga);
        c.ar.reset_tmp();
      }
      const GatedW& g = W.bond[t];
      float* g_agg = c.f(false, (size_t)Es * 64);
      lin(g_e, b.short_ids, Es, 64, g.wo, nullptr, nullptr, nullptr, 64, g_agg);
      float* g_pre = c.f(false, (size_t)A * 128);
      float *gw_i = c.f(false, (size_t)A * 64), *gw_j = c.f(false, (size_t)A * 64);
      RUN(c, "bond_conv_bwd", chg_bond_conv_bwd(sb[t].pre, sb[t].p, wbg_s, b.ang_is, b.ang_js, A, g_agg, g.w2, g.ln, g_pre, gw_i,
                                                gw_j, nullptr, nullptr, st));
      lin(g_pre, nullptr, A, 128, g.c_b, nullptr, g_a_live ? g_a : nullptr, nullptr, 64, g_a);
      g_a_live = true;
      angle_scatter(g_pre, g);
      seg(gw_i, 64, nullptr, b.ptr_is, Es, A, 1, g_wbg, 64);
      seg(gw_j, 64, b.perm_js, b.ptr_js, Es, A, 1, g_wbg, 64);
      c.ar.reset_tmp();
    }
    atom_bwd(t);
  }

  float* g_dist = c.f(false, Eu);
  float* g_wbg_full = c.f(false, (size_t)Eu * 64);
  c.zero(g_wbg_full, (size_t)Eu * 256);
  if (has_ang) RUN(c, "scatter_rows", chg_scatter_rows(g_wbg, b.short_ids, Es, 64, g_wbg_full, st));
  RUN(c, "bond_basis_bwd", chg_bond_basis_bwd(dist, b.u2d, Eu, W.freq_ag, W.freq_bg, hp.num_radial, hp.atom_graph_cutoff,
                                              hp.bond_graph_cutoff, hp.cutoff_coeff, W.w3, g_e, g_wag, g_wbg_full, g_dist, nullptr, st));
  double* g_rhat = static_cast<double*>(c.ar.tmp((size_t)Ed * 3 * 8));
  c.zero(g_rhat, (size_t)Ed * 24);
  // with one block no BondConv reverse ran: the angle features feed nothing, dE/d(angle basis) = 0 and g_rhat stays zero
  if (has_ang && g_a_live)
    RUN(c, "angle_basis_bwd", chg_angle_basis_bwd(rhat, b.ang_di, b.ang_dj, A, W.freq_ang, (hp.num_angular - 1) / 2, W.wang, g_a,
                                                  g_rhat, nullptr, st));
  c.zero(o.force, (size_t)N * 24);
  c.zero(o.virial, (size_t)B * 72);
  RUN(c, "force_virial", chg_force_virial(rvec, dist, rhat, g_rhat, g_dist, b.d2u, b.u2d, b.center, b.nbr, b.owner, Ed, o.force,
                                          o.virial, st));
  c.ar.reset_tmp();
  return c.rc;
}

}  // namespace
}  // namespace chg

using namespace chg;

extern "C" int64_t chg_packed_floats(const chg_hparams* hp) {
  if (!hp_ok(hp)) return -1;
  Weights w;
  return walk(*hp, nullptr, w);
}

extern "C" int chg_pack_weights_host(chg_hparams* hp, const chg_state_dict* sd, float* packed) {
  CHG_CHECK_ARG(hp_ok(hp), "bad hyper-parameters");
  CHG_CHECK_ARG(sd != nullptr && packed != nullptr, "null pointer");
  Weights w;
  const int64_t total = walk(*hp, packed, w);
  std::memset(packed, 0, sizeof(float) * total);
  const int R = hp->num_radial, NA = hp->num_angular, F = (NA - 1) / 2, L = hp->n_readout_hidden;
  copy_n(w.emb, sd->atom_embedding, 94 * 64);
  copy_n(w.freq_ag, sd->freq_ag, R);
  copy_n(w.freq_bg, sd->freq_bg, R);
  copy_n(w.freq_ang, sd->freq_ang, F);
  const float* three[3] = {sd->bond_embedding, sd->bond_weights_ag, sd->bond_weights_bg};
  for (int m = 0; m < 3; ++m) {
    copy_n(w.w3 + (size_t)m * 64 * R, three[m], 64 * R);
    for (int o = 0; o < 64; ++o)
      for (int k = 0; k < R; ++k) mut(w.w3t)[((size_t)m * R + k) * 64 + o] = three[m][(size_t)o * R + k];
  }
  copy_n(w.wang, sd->angle_embedding, 64 * NA);
  for (int o = 0; o < 64; ++o)
    for (int k = 0; k < NA; ++k) mut(w.wang_t)[(size_t)k * 64 + o] = sd->angle_embedding[(size_t)o * NA + k];
  for (int t = 0; t < hp->n_conv; ++t) {  // AtomConv first layer [64][192] = [centre | bond | neighbour]
    const GatedW& g = w.atom[t];
    const chg_gated_sd& s = sd->atom[t];
    pack_second(g, s);
    pack_ln(g, s);
    put_t(g.a_t, 256, 0, s.core_w1, 192, 0);
    put_t(g.a_t, 256, 64, s.gate_w1, 192, 0);
    put_t(g.a_t, 256, 128, s.core_w1, 192, 128);
    put_t(g.a_t, 256, 192, s.gate_w1, 192, 128);
    put_t(g.b_t, 128, 0, s.core_w1, 192, 64);
    put_t(g.b_t, 128, 64, s.gate_w1, 192, 64);
    copy_n(g.bias1, s.core_b1, 64);
    copy_n(g.bias1 + 64, s.gate_b1, 64);
    put_rows(g.a_b, 0, s.core_w1, 192, 0);
    put_rows(g.a_b, 1, s.gate_w1, 192, 0);
    put_rows(g.a_b, 2, s.core_w1, 192, 128);
    put_rows(g.a_b, 3, s.gate_w1, 192, 128);
    put_rows(g.b_b, 0, s.core_w1, 192, 64);
    put_rows(g.b_b, 1, s.gate_w1, 192, 64);
    pack_out(g, s);
  }
  for (int t = 0; t < hp->n_conv - 1; ++t) {  // BondConv / AngleUpdate first layer [64][256] = [bond i | bond j | angle | centre]
    for (int kind = 0; kind < 2; ++kind) {
      const GatedW& g = kind == 0 ? w.bond[t] : w.angle[t];
      const chg_gated_sd& s = kind == 0 ? sd->bond[t] : sd->angle[t];
      if (kind == 0) pack_second(g, s);
      pack_ln(g, s);
      put_t(g.a_t, 256, 0, s.core_w1, 256, 0);
      put_t(g.a_t, 256, 64, s.gate_w1, 256, 0);
      put_t(g.a_t, 256, 128, s.core_w1, 256, 64);
      put_t(g.a_t, 256, 192, s.gate_w1, 256, 64);
      copy_n(g.bias1, s.core_b1, 64);
      copy_n(g.bias1 + 64, s.gate_b1, 64);
      put_t(g.b_t, 128, 0, s.core_w1, 256, 192);
      put_t(g.b_t, 128, 64, s.gate_w1, 256, 192);
      put_t(g.c_t, 128, 0, s.core_w1, 256, 128);
      put_t(g.c_t, 128, 64, s.gate_w1, 256, 128);
      put_rows(g.a_b, 0, s.core_w1, 256, 0);
      put_rows(g.a_b, 1, s.gate_w1, 256, 0);
      put_rows(g.a_b, 2, s.core_w1, 256, 64);
      put_rows(g.a_b, 3, s.gate_w1, 256, 64);
      put_rows(g.b_b, 0, s.core_w1, 256, 192);
      put_rows(g.b_b, 1, s.gate_w1, 256, 192);
      put_rows(g.c_b, 0, s.core_w1, 256, 128);
      put_rows(g.c_b, 1, s.gate_w1, 256, 128);
      if (kind == 0) pack_out(g, s);
    }
  }
  if (w.readout_ln != nullptr) {
    copy_n(w.readout_ln, sd->readout_ln_w, 64);
    copy_n(w.readout_ln + 64, sd->readout_ln_b, 64);
  }
  for (int l = 0; l < L; ++l) {
    copy_n(w.mlp_w + (size_t)l * 4096, sd->mlp_w[l], 4096);
    put_t(w.mlp_wt + (size_t)l * 4096, 64, 0, sd->mlp_w[l], 64, 0);
    copy_n(w.mlp_b + (size_t)l * 64, sd->mlp_b[l], 64);
  }
  copy_n(w.w_last, sd->mlp_last_w, 64);
  copy_n(w.w_mag, sd->site_wise_w, 64);
  if (sd->atom_ref != nullptr) copy_n(w.atom_ref, sd->atom_ref, 94);
  hp->b_last = sd->mlp_last_b;
  hp->b_mag = sd->site_wise_b;
  return CHG_OK;
}

static int forward_impl(const chg_hparams* hp, const float* packed, const chg_batch* b, const chg_outputs* o, void* workspace,
                        size_t workspace_bytes, bool dry, std::string* trace, size_t* need, void* stream) {
  CHG_CHECK_ARG(hp_ok(hp), "bad hyper-parameters");
  CHG_CHECK_ARG(b != nullptr && o != nullptr, "null pointer");
  CHG_CHECK_ARG(b->n_atoms >= 0 && b->n_edges >= 0 && b->n_bonds >= 0 && b->n_angles >= 0 && b->n_graphs >= 1 && b->n_short >= 0,
                "negative size");
  Weights w;
  walk(*hp, const_cast<float*>(packed), w);
  Ctx c;
  c.ar.base = static_cast<char*>(workspace);
  c.ar.cap = dry ? (size_t)-1 / 4 : workspace_bytes / ALIGN * ALIGN;
  c.ar.dry = dry;
  c.stream = as_stream(stream);
  c.trace = trace;
  const int rc = run_schedule(*hp, w, *b, *o, c);
  if (need != nullptr) *need = c.ar.peak + ALIGN;
  if (!dry && c.ar.overflow) {
    set_error("chg_forward: workspace too small (%zu bytes given, %zu needed; ask chg_forward_plan)", workspace_bytes,
              c.ar.peak + ALIGN);
    return CHG_ERR_ARG;
  }
  return rc;
}

extern "C" int chg_forward_plan(const chg_hparams* hp, const chg_batch* sizes, const chg_outputs* wanted,
                                size_t* workspace_bytes, char* trace, size_t trace_cap) {
  std::string tr;
  const int rc = forward_impl(hp, nullptr, sizes, wanted, nullptr, 0, true, trace != nullptr ? &tr : nullptr, workspace_bytes, nullptr);
  if (trace != nullptr && trace_cap > 0) {
    const size_t n = tr.size() < trace_cap - 1 ? tr.size() : trace_cap - 1;
    std::memcpy(trace, tr.data(), n);
    trace[n] = 0;
  }
  return rc;
}

extern "C" int chg_forward(const chg_hparams* hp, const float* packed_weights, const chg_batch* batch, const chg_outputs* out,
                           void* workspace, size_t workspace_bytes, void* stream) {
  CHG_CHECK_ARG(packed_weights != nullptr && workspace != nullptr, "null pointer");
  CHG_CHECK_ARG(out != nullptr && out->energy && out->e_ref && out->site_e, "energy, e_ref and site_e outputs are required");
  CHG_CHECK_ARG(((uintptr_t)workspace & (ALIGN - 1)) == 0 && ((uintptr_t)packed_weights & 63) == 0,
                "workspace must be 256-byte aligned, packed_weights 64-byte aligned");
  return forward_impl(hp, packed_weights, batch, out, workspace, workspace_bytes, false, nullptr, nullptr, stream);
}
