"""Kernel schedule of the hot path: forward, then ONE reverse pass for F and sigma.

Restates what ``CHGNet._compute`` does (reference chgnet/model/model.py:389-542)
as a fixed sequence of C-ABI kernel calls on a :class:`DeviceBatch`:

    geometry/basis/embeddings -> 3 x (AtomConv, BondConv, AngleUpdate) -> AtomConv
    -> readout  [-> reverse of all of it -> force / virial]

Differences from the reference that are deliberate (DESIGN.md §3):
* the dead third AngleUpdate (its output is never read, model.py:470-496) is skipped;
* forces and stress come from one reverse pass producing dE/dr per directed
  edge (the reference runs autograd twice, model.py:521-535);
* no ``create_graph=True`` in inference;
* every scatter-add is a segmented reduction over the batch's CSR structures.

``kernels`` is the binding object (``chgnet_b200._lib.CudaKernels``).  There is no
CPU implementation in the product: constructing the engine without the CUDA
library raises.  Tests inject ``oracle.kernel_specs.SpecKernels`` to check this
schedule on the CPU.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import torch
from torch import Tensor

from chgnet_b200.batch import DeviceBatch
from chgnet_b200.weights import PackedWeights

EV_A3_TO_GPA = 160.21766208  # reference model.py:533


@dataclass
class EngineOutput:
    energy: Tensor  # [B] fp64 model energy (extensive, eV)
    e_ref: Tensor  # [B] fp64 AtomRef energy (extensive)
    site_e: Tensor  # [N]
    magmom: Tensor | None = None
    atom_fea: Tensor | None = None
    crystal_fea: Tensor | None = None
    force: Tensor | None = None  # [N,3] fp64
    virial: Tensor | None = None  # [B,9] fp64, sum_e r (x) dE/dr
    extras: dict = field(default_factory=dict)


class Engine:
    def __init__(self, pw: PackedWeights, kernels) -> None:
        if kernels is None:
            raise RuntimeError("chgnet_b200 Engine needs the CUDA kernel library (no CPU path exists)")
        self.pw = pw
        self.K = kernels

    # ------------------------------------------------------------------ helpers
    def _new(self, b: DeviceBatch, *shape, dtype=None) -> Tensor:
        return torch.empty(*shape, dtype=dtype or self.pw.emb.dtype, device=b.z.device)

    def _zeros(self, b: DeviceBatch, *shape, dtype=None) -> Tensor:
        return torch.zeros(*shape, dtype=dtype or self.pw.emb.dtype, device=b.z.device)

    def _lin(self, b, x, wt, bias=None, residual=None, x_rows=None) -> Tensor:
        m = x.shape[0] if x_rows is None else x_rows.shape[0]
        y = self._new(b, m, wt.shape[1])
        self.K.linear(x, wt, bias, residual, y, x_rows, None)
        return y

    def _seg(self, b, data, perm, ptr, n_rows) -> Tensor:
        out = self._new(b, n_rows, data.shape[1])
        self.K.segment_sum(data, perm, ptr, 0, out)
        return out

    # ------------------------------------------------------------------ forward (+ reverse)
    def run(
        self,
        b: DeviceBatch,
        *,
        need_grad: bool,
        need_magmom: bool = False,
        need_atom_fea: bool = False,
        need_crystal_fea: bool = False,
        keep_intermediates: bool = False,
        train: bool = False,
    ) -> EngineOutput:
        """Forward; with ``need_grad`` the reverse pass for F / sigma right after it.

        ``train=True`` (reference trainer.py:398-411) saves what the PARAMETER gradients need and
        returns without a reverse pass: call :meth:`param_grads` with the loss seeds afterwards.
        """
        pw, K, hp = self.pw, self.K, self.pw.hp
        if train:
            need_grad = True
        N, Ed, Eu, A, B = b.n_atoms, b.n_edges, b.n_bonds, b.n_angles, b.n_graphs
        has_ang = A > 0
        n_conv = hp.n_conv
        inter: dict = {}

        # ---- geometry, bases, embeddings -------------------------------------
        x = self._new(b, N, 64)
        K.embed_atoms(b.z, pw.emb, x)
        rvec, dist, rhat = self._new(b, Ed, 3), self._new(b, Ed), self._new(b, Ed, 3)
        K.edge_geometry(b.frac, b.lattice, b.owner, b.center, b.nbr, b.image, rvec, dist, rhat)
        e, wag, wbg = self._new(b, Eu, 64), self._new(b, Eu, 64), self._new(b, Eu, 64)
        tr: dict = dict(x=[], e=[], ang=[], agg_a=[], agg_b=[]) if train else {}
        if train:
            tr["bb"] = self._new(b, Eu, 64)
            K.bond_basis_embed(dist, b.u2d, pw.freq_ag, pw.freq_bg, hp.atom_graph_cutoff, hp.bond_graph_cutoff,
                               hp.cutoff_coeff, pw.w3t, e, wag, wbg, tr["bb"])
        else:
            K.bond_basis_embed(dist, b.u2d, pw.freq_ag, pw.freq_bg, hp.atom_graph_cutoff, hp.bond_graph_cutoff,
                               hp.cutoff_coeff, pw.w3t, e, wag, wbg)
        ang = None
        if has_ang:
            ang = self._new(b, A, 64)
            if train:
                tr["fb"] = self._new(b, A, 64)
                K.angle_basis_embed(rhat, b.ang_di, b.ang_dj, pw.freq_ang, pw.wang_t, ang, tr["fb"])
            else:
                K.angle_basis_embed(rhat, b.ang_di, b.ang_dj, pw.freq_ang, pw.wang_t, ang)
        if keep_intermediates:
            inter.update(x0=x, e0=e, w_ag=wag, w_bg=wbg, a0=ang)

        saved_atom: list[dict] = []
        saved_bond: list[dict] = []
        saved_angle: list[dict] = []

        def atom_conv(t: int, x: Tensor, e: Tensor) -> Tensor:
            gp = pw.atom[t]
            pcn = self._lin(b, x, gp.extra["wcn_t"])
            pe = self._lin(b, e, gp.extra["we_t"], bias=gp.extra["b1"])
            save_p = self._new(b, Ed, 128) if need_grad else None
            agg = self._new(b, N, 64)
            if train:  # training also keeps `pre` and the message: unfused pair
                msg = self._new(b, Ed, 64)
                save_pre = self._new(b, Ed, 128)
                K.atom_conv_fwd(pcn, pe, wag, b.center, b.nbr, b.d2u, gp.w2t, gp.b2, gp.ln, msg, save_p, save_pre)
                K.segment_sum(msg, None, b.ptr_c, 0, agg)
            else:  # message + aggregation in one kernel: the [Ed, 64] message never reaches HBM
                K.atom_conv_fused(pcn, pe, wag, b.center, b.nbr, b.d2u, b.ptr_c, gp.w2t, gp.b2, gp.ln, agg, save_p)
            if need_grad:
                saved_atom.append(dict(pcn=pcn, pe=pe, p=save_p))
            if train:
                saved_atom[-1].update(pre=save_pre, x=x, e=e, agg=agg)
            return self._lin(b, agg, gp.extra["wo_t"], bias=gp.extra["bo"], residual=x)

        # BondConv / AngleUpdate work in the compact space of the Es bond-graph bonds
        Es, sid = b.n_short, b.short_ids
        wbg_s = None
        if has_ang:
            wbg_s = self._new(b, Es, 64)
            K.gather_rows(wbg, sid, wbg_s)

        magmom = atom_fea = None
        for t in range(n_conv - 1):
            x = atom_conv(t, x, e)
            if has_ang:
                gp = pw.bond[t]
                pij = self._lin(b, e, gp.extra["wij_t"], bias=gp.extra["bij"], x_rows=sid)
                px = self._lin(b, x, gp.extra["wx_t"])
                pa = self._lin(b, ang, gp.extra["w1a_t"])  # angle block of the first layer, per angle
                s_pre = self._new(b, A, 128) if need_grad else None
                s_p = self._new(b, A, 128) if need_grad else None
                agg = self._new(b, Es, 64)
                if train:
                    upd = self._new(b, A, 64)
                    K.bond_conv_fwd(pij, px, pa, wbg_s, b.ang_atom, b.ang_is, b.ang_js, gp.w2t, gp.b2, gp.ln,
                                    upd, s_pre, s_p)
                    K.segment_sum(upd, None, b.ptr_is, 0, agg)
                else:
                    K.bond_conv_fused(pij, px, pa, wbg_s, b.ang_atom, b.ang_is, b.ang_js, b.ptr_is, gp.w2t, gp.b2, gp.ln,
                                      agg, s_pre, s_p)
                # e[sid] += Wo agg (+ bias); bonds outside the bond graph keep their features
                # (with mlp_out bias the batch is built with identity compaction, Es == Eu)
                e_in = e
                if keep_intermediates or train:
                    e = e.clone()
                K.linear(agg, gp.extra["wo_t"], gp.extra["bo"], e, e, None, sid)
                if need_grad:
                    saved_bond.append(dict(pre=s_pre, p=s_p))
                if train:
                    saved_bond[-1].update(x=x, e=e_in, ang=ang, agg=agg)
                if t < n_conv - 2:  # the last AngleUpdate is dead compute
                    ga = pw.angle[t]
                    pij = self._lin(b, e, ga.extra["wij_t"], bias=ga.extra["bij"], x_rows=sid)
                    px = self._lin(b, x, ga.extra["wx_t"])
                    pa = self._lin(b, ang, ga.extra["w1a_t"])
                    ang_new = self._new(b, A, 64)
                    s_p = self._new(b, A, 128) if need_grad else None
                    K.angle_update_fwd(pij, px, pa, ang, b.ang_atom, b.ang_is, b.ang_js, ga.ln, ang_new, s_p)
                    if need_grad:
                        saved_angle.append(dict(p=s_p))
                    if train:
                        saved_angle[-1].update(x=x, e=e, ang=ang)
                    ang = ang_new
            if keep_intermediates:
                inter[f"x{t + 1}"], inter[f"e{t + 1}"] = x, e
                if t < n_conv - 2:
                    inter[f"a{t + 1}"] = ang
            if t == n_conv - 2:  # model.py:477-487
                if need_atom_fea:
                    atom_fea = x
                if need_magmom:
                    magmom = self._new(b, N)
                    K.magmom(x, pw.w_mag, pw.b_mag, magmom)
                    tr["x_mag"] = x
        x = atom_conv(n_conv - 1, x, e)

        # ---- readout -----------------------------------------------------------
        site_e = self._new(b, N)
        h_out = self._new(b, N, 64) if (need_crystal_fea or keep_intermediates) else None
        energy = self._zeros(b, B, dtype=torch.float64)
        e_ref = self._zeros(b, B, dtype=torch.float64)
        g_x = self._new(b, N, 64) if need_grad else None
        K.readout(x, b.z, b.owner, pw.readout_ln, pw.mlp_wt, pw.mlp_w, pw.mlp_b, pw.w_last, pw.b_last,
                  pw.atom_ref, site_e, h_out, energy, e_ref, g_x)
        crystal_fea = None
        if need_crystal_fea:
            gptr = torch.zeros(B + 1, dtype=torch.int32, device=b.z.device)
            gptr[1:] = torch.cumsum(torch.tensor(b.atoms_per_graph, device=b.z.device), 0)
            crystal_fea = self._seg(b, h_out, None, gptr, B)
        if keep_intermediates:
            inter["x_readout"], inter["site_e_model"] = h_out, site_e
        out = EngineOutput(energy=energy, e_ref=e_ref, site_e=site_e, magmom=magmom, atom_fea=atom_fea,
                           crystal_fea=crystal_fea, extras=inter)
        if not need_grad:
            return out
        st = dict(b=b, x_last=x, g_x=g_x, wag=wag, wbg_s=wbg_s, dist=dist, rvec=rvec, rhat=rhat, tr=tr,
                  saved_atom=saved_atom, saved_bond=saved_bond, saved_angle=saved_angle)
        if train:
            out.extras["train_state"] = st
            return out
        self._reverse(st, out, None)
        return out

    # ------------------------------------------------------------------ reverse
    def input_grads(self, out: EngineOutput, record: bool = False) -> None:
        """Forces / virial of a ``train=True`` forward (values only; the state is kept for
        :meth:`param_grads`).  ``record=True`` also keeps the adjoints dE/d(intermediate) that the
        second-order pass of a force / stress loss needs."""
        st = out.extras["train_state"]
        n = self.pw.hp.n_conv
        rec = dict(atom=[None] * n, bond=[None] * (n - 1), angle=[None] * (n - 1)) if record else None
        self._reverse(st, out, None, rec)
        if record:
            st["rec"] = rec

    def param_grads(self, out: EngineOutput, seed_energy: Tensor, seed_magmom: Tensor | None = None,
                    seed_force: Tensor | None = None, seed_stress: Tensor | None = None) -> dict:
        """Training reverse pass (replaces ``loss.backward()``, trainer.py:409-410) for losses on the
        energies and magnetic moments: dL/d(parameter) for ``seed_energy[g] = dL/d(E_g)`` (E_g the
        extensive model energy of graph g) and ``seed_magmom[i] = dL/d(m_i)``.

        Returns gradients in the packed layouts, keyed like ``weights.unpack_grads`` expects.  Losses on
        forces / stresses need the second-order pass (reverse of this reverse pass), which is not
        built yet (DESIGN.md §9); asking for them raises in ``chgnet_b200.trainer``.
        """
        st = out.extras.pop("train_state")
        grads: dict = {}
        if seed_force is not None or seed_stress is not None:
            if "rec" not in st:
                raise RuntimeError("call input_grads(out, record=True) before param_grads with force / stress seeds")
            self._second_order(st, dict(seed_energy=seed_energy, seed_magmom=seed_magmom, seed_force=seed_force,
                                        seed_stress=seed_stress, grads=grads))
            return grads
        self._reverse(st, out, dict(seed_energy=seed_energy, seed_magmom=seed_magmom, grads=grads))
        return grads

    def hessian_vector_products(self, b: DeviceBatch, directions: Tensor) -> Tensor:
        """H v per atom, ``[N,3]`` fp64, H = d^2E/dx dx of the extensive model energy of each graph (cell fixed,
        x Cartesian positions), v = ``directions`` ``[N,3]``.  A batch of K copies of one graph with a different
        direction on each copy gives K products of that graph's Hessian in one call."""
        out = self.run(b, need_grad=True, train=True)
        self.input_grads(out, record=True)
        st = out.extras.pop("train_state")
        return self._second_order(st, dict(seed_energy=self._zeros(b, b.n_graphs, dtype=torch.float64), seed_magmom=None,
                                           seed_force=None, seed_stress=None, grads=None, directions=directions))[0]

    def second_derivatives(self, b: DeviceBatch, directions: Tensor, strain_directions: Tensor) -> tuple[Tensor, Tensor]:
        """dT/dx per atom ``[N,3]`` and dT/d(strain) per graph ``[B,3,3]``, both fp64, for
        T = <dE/dx, v> + <dE/dstrain, W> of each graph: v = ``directions`` ``[N,3]``, W = ``strain_directions``
        ``[B,3,3]``.  Strain maps every edge vector r_e -> r_e (I + strain) (fractional coordinates fixed), so
        dE/dstrain = sum_e r_e (x) dE/dr_e; E is the extensive model energy.  The two outputs are
        H v + Lambda W and Lambda^T v + D W, with H = d^2E/dx dx, D = d^2E/dstrain dstrain and Lambda the
        position-strain block d^2E/dx dstrain, all second derivatives of E(r) taken through the edge vectors with
        rdot_e = v[c] - v[n] + r_e . W held fixed (for Lambda: -dF/dstrain at fixed fractional coordinates)."""
        out = self.run(b, need_grad=True, train=True)
        self.input_grads(out, record=True)
        st = out.extras.pop("train_state")
        hv, dt_dstrain = self._second_order(st, dict(
            seed_energy=self._zeros(b, b.n_graphs, dtype=torch.float64), seed_magmom=None, seed_force=None,
            seed_stress=None, grads=None, directions=directions, strain_directions=strain_directions))
        return hv, dt_dstrain.view(b.n_graphs, 3, 3)

    # ------------------------------------------------------------------ second order
    def _second_order(self, st: dict, train: dict) -> tuple[Tensor, Tensor] | None:
        """Parameter gradients of a loss that also depends on forces and stresses (reference
        model.py:518-535 ``create_graph=True`` + trainer.py:409 ``loss.backward()``).

        With F = -dE/dcart and sigma = (c/V) dE/d(strain), the force / stress part of the loss gradient is
        d/dtheta of  T = sum_e <dE/dr_e, rdot_e>,  rdot_e = -(gF[c] - gF[n]) + r_e . (gS c/V)  held fixed.
        T is evaluated by a TANGENT pass (forward mode along rdot through every kernel of the forward
        pass), and differentiated by one more reverse pass over (primal, tangent).  The adjoint of every
        tangent quantity equals the ordinary adjoint lambda = dE/d(.) recorded by the force pass, so this
        reverse pass only propagates the adjoints of the PRIMAL intermediates ("bar"), seeded with the
        energy / magmom loss, and adds the second-order source terms inside the nonlinear kernels.

        Hessian-vector mode (``train["grads"] is None``, ``train["directions"]`` = v per atom, zero energy seed):
        rdot_e = v[c] - v[n], so T = <dE/dx, v>, and dT/dx = H v.  No parameter gradient is formed; the tail
        differentiates T with respect to the geometry instead (:meth:`_geometry_tail`) and returns H v.  With
        ``train["strain_directions"]`` = W per graph as well, rdot_e gains r_e . W and the tail also returns the
        per-graph strain derivative of T (:meth:`second_derivatives`).
        """
        pw, K, hp = self.pw, self.K, self.pw.hp
        b: DeviceBatch = st["b"]
        N, Ed, Eu, A, B = b.n_atoms, b.n_edges, b.n_bonds, b.n_angles, b.n_graphs
        has_ang = A > 0
        n_conv = hp.n_conv
        Es, sid = b.n_short, b.short_ids
        wag, wbg_s, dist, rvec, rhat, tr, rec = st["wag"], st["wbg_s"], st["dist"], st["rvec"], st["rhat"], st["tr"], st["rec"]
        saved_atom, saved_bond, saved_angle = st["saved_atom"], st["saved_bond"], st["saved_angle"]
        G = train["grads"]
        dt = pw.emb.dtype
        use_ln = pw.atom[0].ln is not None

        def ln_acc():
            return self._zeros(b, 256, dtype=torch.float64) if (G is not None and use_ln) else None

        def lin(x, wt, residual=None, x_rows=None):
            return self._lin(b, x, wt, None, residual, x_rows)

        def wsum(x, g, n, xd, lam, **kw):
            """x^T g + xd^T lam : weight gradient of a linear op and of its tangent"""
            return self._wgrad(b, x, g, n, **kw) + self._wgrad(b, xd, lam, n, **kw)

        # ---------------- tangent pass ----------------
        if train.get("directions") is not None:
            u_atom = train["directions"].to(dt).contiguous()
        elif train["seed_force"] is not None:
            u_atom = (-train["seed_force"]).to(dt).contiguous()
        else:
            u_atom = self._zeros(b, N, 3)
        w_graph = self._zeros(b, B, 9)
        if train["seed_stress"] is not None:
            scale = (EV_A3_TO_GPA / b.volume.to(torch.float64))[:, None, None]
            w_graph = (train["seed_stress"].to(torch.float64).view(B, 3, 3) * scale).to(dt).reshape(B, 9).contiguous()
        per_graph = train.get("strain_directions") is not None
        if per_graph:
            w_graph = train["strain_directions"].to(dt).reshape(B, 9).contiguous()
        ddist, drhat = self._new(b, Ed), self._new(b, Ed, 3)
        K.edge_tangent(rvec, dist, rhat, b.center, b.nbr, b.owner, u_atom, w_graph, ddist, drhat)
        e_d, wag_d, wbg_d, tb = (self._new(b, Eu, 64) for _ in range(4))
        K.bond_basis_tangent(dist, ddist, b.u2d, pw.freq_ag, pw.freq_bg, hp.atom_graph_cutoff, hp.bond_graph_cutoff,
                             hp.cutoff_coeff, pw.w3t, e_d, wag_d, wbg_d, tb)
        ang_d = tfb = wbg_s_d = None
        if has_ang:
            ang_d, tfb = self._new(b, A, 64), self._new(b, A, 64)
            K.angle_basis_tangent(rhat, drhat, b.ang_di, b.ang_dj, pw.freq_ang, pw.wang_t, ang_d, tfb)
            wbg_s_d = self._new(b, Es, 64)
            K.gather_rows(wbg_d, sid, wbg_s_d)
        x_d = self._zeros(b, N, 64)
        t_atom, t_bond, t_angle = [None] * n_conv, [None] * (n_conv - 1), [None] * (n_conv - 1)

        def atom_tan(t, x_d, e_d):
            gp, sv = pw.atom[t], saved_atom[t]
            pcn_d, pe_d = lin(x_d, gp.extra["wcn_t"]), lin(e_d, gp.extra["we_t"])
            msg_d, pre_d, p_d = self._new(b, Ed, 64), self._new(b, Ed, 128), self._new(b, Ed, 128)
            K.atom_conv_tan(pcn_d, pe_d, wag, wag_d, b.center, b.nbr, b.d2u, sv["pre"], sv["p"], gp.w2t, gp.ln,
                            msg_d, pre_d, p_d)
            agg_d = self._seg(b, msg_d, None, b.ptr_c, N)
            t_atom[t] = dict(x_d=x_d, e_d=e_d, pre_d=pre_d, p_d=p_d, agg_d=agg_d)
            return lin(agg_d, gp.extra["wo_t"], residual=x_d)

        for t in range(n_conv - 1):
            x_d = atom_tan(t, x_d, e_d)
            if has_ang:
                gp, sv = pw.bond[t], saved_bond[t]
                pij_d = lin(e_d, gp.extra["wij_t"], x_rows=sid)
                px_d, pa_d = lin(x_d, gp.extra["wx_t"]), lin(ang_d, gp.extra["w1a_t"])
                upd_d, pre_d, p_d = self._new(b, A, 64), self._new(b, A, 128), self._new(b, A, 128)
                K.bond_conv_tan(pij_d, px_d, pa_d, wbg_s, wbg_s_d, b.ang_atom, b.ang_is, b.ang_js, sv["pre"], sv["p"],
                                gp.w2t, gp.ln, upd_d, pre_d, p_d)
                agg_d = self._seg(b, upd_d, None, b.ptr_is, Es)
                t_bond[t] = dict(x_d=x_d, e_d=e_d, ang_d=ang_d, pre_d=pre_d, p_d=p_d, agg_d=agg_d)
                e_d = e_d.clone()
                K.linear(agg_d, gp.extra["wo_t"], None, e_d, e_d, None, sid)
                if t < n_conv - 2:
                    ga, sva = pw.angle[t], saved_angle[t]
                    pij_d = lin(e_d, ga.extra["wij_t"], x_rows=sid)
                    px_d, pa_d = lin(x_d, ga.extra["wx_t"]), lin(ang_d, ga.extra["w1a_t"])
                    ang_new_d, p_d = self._new(b, A, 64), self._new(b, A, 128)
                    K.angle_update_tan(pij_d, px_d, pa_d, ang_d, b.ang_atom, b.ang_is, b.ang_js, sva["p"], ga.ln,
                                       ang_new_d, p_d)
                    t_angle[t] = dict(x_d=x_d, e_d=e_d, ang_d=ang_d, p_d=p_d)
                    ang_d = ang_new_d
        x_d = atom_tan(n_conv - 1, x_d, e_d)

        # ---------------- reverse over (primal, tangent) ----------------
        L = pw.mlp_wt.shape[0]
        seed_atom = train["seed_energy"].to(dt)[b.owner.long()].contiguous()
        bar_x = self._new(b, N, 64)
        h_all, hd_all = self._new(b, L + 1, N, 64), self._new(b, L + 1, N, 64)
        gz_all, zbar_all = self._new(b, L, N, 64), self._new(b, L, N, 64)
        g_h0, hbar0, xhat, xhatd = (self._new(b, N, 64) for _ in range(4))
        K.readout_bwd2(st["x_last"], x_d, pw.readout_ln, pw.mlp_wt, pw.mlp_w, pw.mlp_b, pw.w_last, seed_atom, bar_x,
                       h_all, hd_all, gz_all, zbar_all, g_h0, hbar0, xhat, xhatd)
        if G is not None:
            G["mlp_wt"] = torch.stack([wsum(h_all[l], zbar_all[l], 64, hd_all[l], gz_all[l]) for l in range(L)])
            G["mlp_b"] = torch.stack([self._colsum(b, zbar_all[l]) for l in range(L)])
            G["w_last"] = self._colsum(b, h_all[L], rowscale=seed_atom) + self._colsum(b, hd_all[L])
            G["b_last"] = seed_atom.sum()
            if pw.readout_ln is not None:
                G["readout_ln"] = torch.stack([self._colsum(b, hbar0, xhat) + self._colsum(b, g_h0, xhatd),
                                               self._colsum(b, hbar0)])

        bar_e = None
        bar_wag = self._zeros(b, Eu, 64)
        bar_wbg = self._zeros(b, Es, 64) if has_ang else None
        bar_a = None

        def acc(dst, x_in, wt):
            return self._lin(b, x_in, wt, residual=dst)

        def w2_grads(key, pre, u, pre_d, g_p_lam, g_ln):
            if G is None:
                return
            w2t, b2, tmp = self._new(b, 64, 128), self._new(b, 128), self._new(b, 64, 128)
            for h in (slice(0, 64), slice(64, 128)):
                K.wgrad(pre[:, h], u[:, h], w2t[:, h], b2[h], None, None, True)       # silu(pre)^T u
                K.wgrad(pre[:, h], g_p_lam[:, h], tmp[:, h], None, None, None, False, pre_d[:, h])  # hdot^T lambda(p)
            G[f"{key}.w2t"], G[f"{key}.b2"] = w2t + tmp, b2
            if g_ln is not None:
                G[f"{key}.ln"] = g_ln.to(dt).view(4, 64)

        def atom_bwd2(t, bar_xout, bar_e):
            gp, sv, la, tt = pw.atom[t], saved_atom[t], rec["atom"][t], t_atom[t]
            if G is not None:
                G[f"atom.{t}.wo_t"] = wsum(sv["agg"], bar_xout, 64, tt["agg_d"], la["g_xout"])
                if gp.extra["bo"] is not None:
                    G[f"atom.{t}.bo"] = self._colsum(b, bar_xout)
            bar_agg = self._lin(b, bar_xout, gp.extra["wo"])
            bar_pre, bar_w, u, g_ln = self._new(b, Ed, 128), self._new(b, Ed, 64), self._new(b, Ed, 128), ln_acc()
            K.atom_conv_bwd2(sv["pre"], sv["p"], tt["pre_d"], tt["p_d"], la["g_p"], wag, wag_d, b.center, b.d2u,
                             la["g_agg"], bar_agg, gp.w2, gp.ln, bar_pre, bar_w, u, g_ln)
            w2_grads(f"atom.{t}", sv["pre"], u, tt["pre_d"], la["g_p"], g_ln)
            sp = self._new(b, N, 256)
            K.segment_sum(bar_pre, None, b.ptr_c, 0, sp[:, :128])
            K.segment_sum(bar_pre, b.perm_n, b.ptr_n, 0, sp[:, 128:])
            spe = self._seg(b, bar_pre, b.perm_u, b.ptr_u, Eu)
            if G is not None:
                G[f"atom.{t}.wcn_t"] = wsum(sv["x"], sp, 256, tt["x_d"], la["sp"])
                we_bar, G[f"atom.{t}.b1"] = self._wgrad(b, sv["e"], spe, 128, colsum=True)
                G[f"atom.{t}.we_t"] = we_bar + self._wgrad(b, tt["e_d"], la["spe"], 128)
            K.segment_sum(bar_w, b.perm_u, b.ptr_u, 1, bar_wag)
            return acc(bar_xout, sp, gp.extra["wcn_b"]), acc(bar_e, spe, gp.extra["we_b"])

        def angle_scatter2(bar_pre, bar_x, bar_e, ex, key, sv, la, tt):
            sp = self._new(b, Es, 256)
            K.segment_sum(bar_pre, None, b.ptr_is, 0, sp[:, :128])
            K.segment_sum(bar_pre, b.perm_js, b.ptr_js, 0, sp[:, 128:])
            if bar_e is None:
                bar_e = self._zeros(b, Eu, 64)
            K.linear(sp, ex["wij_b"], None, bar_e, bar_e, None, sid)
            spx = self._seg(b, bar_pre, b.perm_x, b.ptr_x, N)
            if G is not None:
                G[f"{key}.wij_t"] = wsum(sv["e"], sp, 256, tt["e_d"], la["sp"], x_rows=sid)
                G[f"{key}.wx_t"] = wsum(sv["x"], spx, 128, tt["x_d"], la["spx"])
                w1a_bar, G[f"{key}.b1"] = self._wgrad(b, sv["ang"], bar_pre, 128, colsum=True)
                G[f"{key}.w1a_t"] = w1a_bar + self._wgrad(b, tt["ang_d"], la["g_pre"], 128)
            return acc(bar_x, spx, ex["wx_b"]), bar_e

        bar_x, bar_e = atom_bwd2(n_conv - 1, bar_x, None)
        if train["seed_magmom"] is not None:
            g_lin = self._new(b, N)
            K.magmom_bwd(tr["x_mag"], pw.w_mag, pw.b_mag, train["seed_magmom"].to(dt).contiguous(), bar_x, g_lin)
            G["w_mag"] = self._colsum(b, tr["x_mag"], rowscale=g_lin)
            G["b_mag"] = g_lin.sum()
        for t in reversed(range(n_conv - 1)):
            if has_ang:
                if t < n_conv - 2:
                    ga, sva, la, tt = pw.angle[t], saved_angle[t], rec["angle"][t], t_angle[t]
                    bar_pre, g_ln = self._new(b, A, 128), ln_acc()
                    K.angle_update_bwd2(sva["p"], tt["p_d"], la["g_ang_in"], bar_a, ga.ln, bar_pre, g_ln)
                    if g_ln is not None:
                        G[f"angle.{t}.ln"] = g_ln.to(dt).view(4, 64)
                    bar_a = acc(bar_a, bar_pre, ga.extra["w1a_b"])
                    bar_x, bar_e = angle_scatter2(bar_pre, bar_x, bar_e, ga.extra, f"angle.{t}", sva, la, tt)
                gp, sv, la, tt = pw.bond[t], saved_bond[t], rec["bond"][t], t_bond[t]
                if bar_e is None:
                    bar_e = self._zeros(b, Eu, 64)
                if G is not None:
                    G[f"bond.{t}.wo_t"] = (self._wgrad(b, sv["agg"], bar_e, 64, g_rows=sid)
                                           + self._wgrad(b, tt["agg_d"], la["g_eout"], 64, g_rows=sid))
                    if gp.extra["bo"] is not None:
                        G[f"bond.{t}.bo"] = self._colsum(b, bar_e)
                bar_agg = self._lin(b, bar_e, gp.extra["wo"], x_rows=sid)
                bar_pre, u, g_ln = self._new(b, A, 128), self._new(b, A, 128), ln_acc()
                bw_i, bw_j = self._new(b, A, 64), self._new(b, A, 64)
                K.bond_conv_bwd2(sv["pre"], sv["p"], tt["pre_d"], tt["p_d"], la["g_p"], wbg_s, wbg_s_d, b.ang_is, b.ang_js,
                                 la["g_agg"], bar_agg, gp.w2, gp.ln, bar_pre, bw_i, bw_j, u, g_ln)
                w2_grads(f"bond.{t}", sv["pre"], u, tt["pre_d"], la["g_p"], g_ln)
                bar_a = acc(bar_a, bar_pre, gp.extra["w1a_b"])
                bar_x, bar_e = angle_scatter2(bar_pre, bar_x, bar_e, gp.extra, f"bond.{t}", sv, la, tt)
                K.segment_sum(bw_i, None, b.ptr_is, 1, bar_wbg)
                K.segment_sum(bw_j, b.perm_js, b.ptr_js, 1, bar_wbg)
            bar_x, bar_e = atom_bwd2(t, bar_x, bar_e)

        bar_wbg_full = self._zeros(b, Eu, 64)
        if has_ang:
            K.scatter_rows(bar_wbg, sid, bar_wbg_full)
        if G is None:
            return self._geometry_tail(st, ddist, drhat, bar_e, bar_wag, bar_wbg_full, bar_a, per_graph)

        # ---------------- embeddings, basis weights, basis frequencies ----------------
        R, NA = pw.freq_ag.shape[0], pw.wang.shape[1]
        order = torch.argsort(b.z.long(), stable=True).int()
        zptr = torch.zeros(95, dtype=torch.int32, device=b.z.device)
        zptr[1:] = torch.cumsum(torch.bincount(b.z.long() - 1, minlength=94), 0)
        G["emb"] = self._new(b, 94, 64)
        K.segment_sum(bar_x, order, zptr, 0, G["emb"])
        bb = tr["bb"]
        G["w3t"] = torch.stack([wsum(bb, bar_e, 64, tb, rec["g_e0"])[:R], wsum(bb, bar_wag, 64, tb, rec["g_wag"])[:R],
                                wsum(bb, bar_wbg_full, 64, tb, rec["g_wbg_full"])[32 : 32 + R]])
        g_freq = self._zeros(b, 2, R, dtype=torch.float64)
        K.bond_basis_bwd(dist, b.u2d, pw.freq_ag, pw.freq_bg, hp.atom_graph_cutoff, hp.bond_graph_cutoff,
                         hp.cutoff_coeff, pw.w3, bar_e, bar_wag, bar_wbg_full, self._new(b, Eu), g_freq)
        K.bond_basis_bwd2(dist, ddist, b.u2d, pw.freq_ag, pw.freq_bg, hp.atom_graph_cutoff, hp.bond_graph_cutoff,
                          hp.cutoff_coeff, pw.w3, rec["g_e0"], rec["g_wag"], rec["g_wbg_full"], g_freq)
        G["freq_ag"], G["freq_bg"] = g_freq[0].to(dt), g_freq[1].to(dt)
        if bar_a is not None:  # None with one block (no angle adjoint, rec["g_a0"] is None too)
            G["wang_t"] = wsum(tr["fb"], bar_a, 64, tfb, rec["g_a0"])[:NA]
            g_fa = self._zeros(b, pw.freq_ang.shape[0], dtype=torch.float64)
            K.angle_basis_bwd(rhat, b.ang_di, b.ang_dj, pw.freq_ang, pw.wang, bar_a, None, g_fa)
            K.angle_basis_bwd2(rhat, drhat, b.ang_di, b.ang_dj, pw.freq_ang, pw.wang, rec["g_a0"], g_fa)
            G["freq_ang"] = g_fa.to(dt)

    def _geometry_tail(self, st, ddist, drhat, bar_e, bar_wag, bar_wbg_full, bar_a,
                       per_graph: bool = False) -> tuple[Tensor, Tensor]:
        """dT/dx (= H v) from the basis-level adjoints of the second reverse pass.  Per directed edge, dT/dr_e is
        (a) the first-order geometry reverse fed with the bar adjoints, (b) lambda . d^2B/dd^2 ddist per bond,
        (c) lambda_a0 . d^2 Fourier(theta) along (drhat_i, drhat_j), and (d) the derivative of the tangent map
        (ddist, drhat)(r_e) with rdot fixed, weighted by the recorded lambda_d, lambda_rhat.  (a)-(c) meet in one
        (g_dist, g_rhat) pair that chg_force_virial turns into -dT/dx; (d) accumulates there too.

        Returns (dT/dx [N,3], virial [B,9]).  The virial sum_e r_e (x) dT/dr_e is dT/dstrain; it holds all four
        terms only with ``per_graph`` (chg_edge_tangent_bwd_virial adds (d)), otherwise (a)-(c)."""
        pw, K, hp = self.pw, self.K, self.pw.hp
        b: DeviceBatch = st["b"]
        rec, dist, rvec, rhat = st["rec"], st["dist"], st["rvec"], st["rhat"]
        g_dist = self._new(b, b.n_bonds)
        K.bond_basis_bwd(dist, b.u2d, pw.freq_ag, pw.freq_bg, hp.atom_graph_cutoff, hp.bond_graph_cutoff,
                         hp.cutoff_coeff, pw.w3, bar_e, bar_wag, bar_wbg_full, g_dist)
        K.bond_basis_hvp(dist, ddist, b.u2d, pw.freq_ag, pw.freq_bg, hp.atom_graph_cutoff, hp.bond_graph_cutoff,
                         hp.cutoff_coeff, pw.w3, rec["g_e0"], rec["g_wag"], rec["g_wbg_full"], g_dist)
        g_rhat = self._zeros(b, b.n_edges, 3, dtype=torch.float64)
        if bar_a is not None:  # None with one block: no angle adjoint
            K.angle_basis_bwd(rhat, b.ang_di, b.ang_dj, pw.freq_ang, pw.wang, bar_a, g_rhat)
            K.angle_basis_hvp(rhat, drhat, b.ang_di, b.ang_dj, pw.freq_ang, pw.wang, rec["g_a0"], g_rhat)
        neg_hv = self._zeros(b, b.n_atoms, 3, dtype=torch.float64)
        virial = self._zeros(b, b.n_graphs, 9, dtype=torch.float64)
        K.force_virial(rvec, dist, rhat, g_rhat, g_dist, b.d2u, b.u2d, b.center, b.nbr, b.owner, neg_hv, virial)
        if per_graph:
            K.edge_tangent_bwd_virial(rvec, dist, rhat, ddist, drhat, rec["g_dist"], rec["g_rhat"], b.d2u, b.u2d,
                                      b.center, b.nbr, b.owner, neg_hv, virial)
        else:
            K.edge_tangent_bwd(dist, rhat, ddist, drhat, rec["g_dist"], rec["g_rhat"], b.d2u, b.u2d, b.center, b.nbr,
                               neg_hv)
        return neg_hv.neg_(), virial

    def _wgrad(self, b, x, g, n, *, x_rows=None, g_rows=None, x_silu=False, colsum=False):
        out = self._new(b, 64, n)
        cs = self._new(b, n) if colsum else None
        self.K.wgrad(x, g, out, cs, x_rows, g_rows, x_silu)
        return (out, cs) if colsum else out

    def _colsum(self, b, a, bmul=None, rowscale=None) -> Tensor:
        out = self._zeros(b, a.shape[1], dtype=torch.float64)
        self.K.colsum(a, out, bmul, rowscale)
        return out.to(self.pw.emb.dtype)

    def _reverse(self, st: dict, out: EngineOutput, train: dict | None, rec: dict | None = None) -> None:
        """``rec`` (inference seeds only): keep the adjoints (lambda = dE/d.) the second-order pass needs."""
        pw, K, hp = self.pw, self.K, self.pw.hp
        b: DeviceBatch = st["b"]
        N, Ed, Eu, A, B = b.n_atoms, b.n_edges, b.n_bonds, b.n_angles, b.n_graphs
        has_ang = A > 0
        n_conv = hp.n_conv
        Es, sid = b.n_short, b.short_ids
        wag, wbg_s, dist, rvec, rhat, tr = st["wag"], st["wbg_s"], st["dist"], st["rvec"], st["rhat"], st["tr"]
        saved_atom, saved_bond, saved_angle = st["saved_atom"], st["saved_bond"], st["saved_angle"]
        G = train["grads"] if train is not None else None
        use_ln = pw.atom[0].ln is not None

        def ln_acc():
            return self._zeros(b, 256, dtype=torch.float64) if (G is not None and use_ln) else None

        g_x = st["g_x"]
        if train is not None:
            # readout reverse with the loss seed, and the readout / magmom parameter gradients
            L = pw.mlp_wt.shape[0]
            seed_atom = train["seed_energy"].to(pw.emb.dtype)[b.owner.long()].contiguous()
            g_x = self._new(b, N, 64)
            h_all, gz_all = self._new(b, L + 1, N, 64), self._new(b, L, N, 64)
            g_h0, xhat = self._new(b, N, 64), self._new(b, N, 64)
            K.readout_bwd(st["x_last"], pw.readout_ln, pw.mlp_wt, pw.mlp_w, pw.mlp_b, pw.w_last, seed_atom, g_x,
                          h_all, gz_all, g_h0, xhat)
            G["mlp_wt"] = torch.stack([self._wgrad(b, h_all[l], gz_all[l], 64) for l in range(L)])
            G["mlp_b"] = torch.stack([self._colsum(b, gz_all[l]) for l in range(L)])
            G["w_last"] = self._colsum(b, h_all[L], rowscale=seed_atom)
            G["b_last"] = seed_atom.sum()
            if pw.readout_ln is not None:
                G["readout_ln"] = torch.stack([self._colsum(b, g_h0, xhat), self._colsum(b, g_h0)])

        g_e = None  # d(sum E)/d e at the current level
        g_wag = self._zeros(b, Eu, 64)
        g_wbg = self._zeros(b, Es, 64) if has_ang else None  # compact; expanded at the end
        g_a = None

        def acc(dst: Tensor | None, x_in: Tensor, wt: Tensor) -> Tensor:
            """dst + x_in @ wt (dst None -> plain product)."""
            return self._lin(b, x_in, wt, residual=dst)

        def w2_grads(key: str, pre: Tensor, g_p: Tensor, g_ln: Tensor | None) -> None:
            """second-layer / LayerNorm parameter gradients of one GatedMLP (block-diagonal core | gate)"""
            w2t, b2 = self._new(b, 64, 128), self._new(b, 128)
            K.wgrad(pre[:, :64], g_p[:, :64], w2t[:, :64], b2[:64], None, None, True)
            K.wgrad(pre[:, 64:], g_p[:, 64:], w2t[:, 64:], b2[64:], None, None, True)
            G[f"{key}.w2t"], G[f"{key}.b2"] = w2t, b2
            if g_ln is not None:
                G[f"{key}.ln"] = g_ln.to(w2t.dtype).view(4, 64)

        def atom_conv_bwd(t: int, g_xout: Tensor, g_e: Tensor | None) -> tuple[Tensor, Tensor]:
            gp, sv = pw.atom[t], saved_atom[t]
            g_agg = self._lin(b, g_xout, gp.extra["wo"])
            g_pre, g_w = self._new(b, Ed, 128), self._new(b, Ed, 64)
            if rec is not None:
                g_p = self._new(b, Ed, 128)
                K.atom_conv_bwd(sv["pcn"], sv["pe"], wag, b.center, b.nbr, b.d2u, sv["p"], g_agg, gp.w2, gp.ln,
                                g_pre, g_w, g_p, None)
                rec["atom"][t] = dict(g_xout=g_xout, g_agg=g_agg, g_p=g_p)
            elif G is None:
                K.atom_conv_bwd(sv["pcn"], sv["pe"], wag, b.center, b.nbr, b.d2u, sv["p"], g_agg, gp.w2, gp.ln,
                                g_pre, g_w)
            else:
                g_p, g_ln = self._new(b, Ed, 128), ln_acc()
                K.atom_conv_bwd(sv["pcn"], sv["pe"], wag, b.center, b.nbr, b.d2u, sv["p"], g_agg, gp.w2, gp.ln,
                                g_pre, g_w, g_p, g_ln)
                w2_grads(f"atom.{t}", sv["pre"], g_p, g_ln)
                G[f"atom.{t}.wo_t"] = self._wgrad(b, sv["agg"], g_xout, 64)
                if gp.extra["bo"] is not None:
                    G[f"atom.{t}.bo"] = self._colsum(b, g_xout)
            sp = self._new(b, N, 256)
            K.segment_sum(g_pre, None, b.ptr_c, 0, sp[:, :128])
            K.segment_sum(g_pre, b.perm_n, b.ptr_n, 0, sp[:, 128:])
            g_xin = acc(g_xout, sp, gp.extra["wcn_b"])
            spe = self._seg(b, g_pre, b.perm_u, b.ptr_u, Eu)
            if rec is not None:
                rec["atom"][t].update(sp=sp, spe=spe)
            if G is not None:
                G[f"atom.{t}.wcn_t"] = self._wgrad(b, sv["x"], sp, 256)
                G[f"atom.{t}.we_t"], G[f"atom.{t}.b1"] = self._wgrad(b, sv["e"], spe, 128, colsum=True)
            g_e = acc(g_e, spe, gp.extra["we_b"])
            K.segment_sum(g_w, b.perm_u, b.ptr_u, 1, g_wag)
            return g_xin, g_e

        def angle_scatter(g_pre: Tensor, g_x: Tensor, g_e: Tensor | None, ex: dict, key: str = "",
                          sv: dict | None = None) -> tuple[Tensor, Tensor]:
            """Push dE/dpre of an angle-indexed GatedMLP back to e (via i and j) and x."""
            sp = self._new(b, Es, 256)
            K.segment_sum(g_pre, None, b.ptr_is, 0, sp[:, :128])
            K.segment_sum(g_pre, b.perm_js, b.ptr_js, 0, sp[:, 128:])
            K.linear(sp, ex["wij_b"], None, g_e, g_e, None, sid)  # g_e[sid] += sp @ Wij
            spx = self._seg(b, g_pre, b.perm_x, b.ptr_x, N)
            if rec is not None:
                rec[key.split(".")[0]][int(key.split(".")[1])].update(sp=sp, spx=spx, g_pre=g_pre)
            if G is not None:  # first-layer blocks: bonds i|j (bias rides on i), centre atom, angle
                G[f"{key}.wij_t"] = self._wgrad(b, sv["e"], sp, 256, x_rows=sid)
                G[f"{key}.wx_t"] = self._wgrad(b, sv["x"], spx, 128)
                G[f"{key}.w1a_t"], G[f"{key}.b1"] = self._wgrad(b, sv["ang"], g_pre, 128, colsum=True)
            g_x = acc(g_x, spx, ex["wx_b"])
            return g_x, g_e

        g_x, g_e = atom_conv_bwd(n_conv - 1, g_x, None)
        if train is not None and train["seed_magmom"] is not None:
            # m = |site_wise(x)| on the output of AtomConv n_conv-2 (model.py:477-487)
            g_lin = self._new(b, N)
            K.magmom_bwd(tr["x_mag"], pw.w_mag, pw.b_mag, train["seed_magmom"].to(pw.emb.dtype).contiguous(), g_x, g_lin)
            G["w_mag"] = self._colsum(b, tr["x_mag"], rowscale=g_lin)
            G["b_mag"] = g_lin.sum()
        for t in reversed(range(n_conv - 1)):
            if has_ang:
                if t < n_conv - 2:  # AngleUpdate_t: a_{t+1} = a_t + G0(e_{t+1}, a_t, x_{t+1})
                    ga = pw.angle[t]
                    g_pre = self._new(b, A, 128)
                    if rec is not None:
                        rec["angle"][t] = dict(g_ang_in=g_a)
                    if G is None:
                        K.angle_update_bwd(saved_angle[t]["p"], g_a, ga.ln, g_pre)
                    else:
                        g_ln = ln_acc()
                        K.angle_update_bwd(saved_angle[t]["p"], g_a, ga.ln, g_pre, g_ln)
                        if g_ln is not None:
                            G[f"angle.{t}.ln"] = g_ln.to(g_pre.dtype).view(4, 64)
                    g_a = acc(g_a, g_pre, ga.extra["w1a_b"])  # residual + through the angle block
                    g_x, g_e = angle_scatter(g_pre, g_x, g_e, ga.extra, f"angle.{t}", saved_angle[t])
                # BondConv_t: e_{t+1} = e_t + Wo agg(G(e_t, a_t, x_{t+1}) w_i w_j)
                gp, sv = pw.bond[t], saved_bond[t]
                g_agg = self._lin(b, g_e, gp.extra["wo"], x_rows=sid)
                g_pre = self._new(b, A, 128)
                gw_i, gw_j = self._new(b, A, 64), self._new(b, A, 64)
                if rec is not None:
                    g_p = self._new(b, A, 128)
                    K.bond_conv_bwd(sv["pre"], sv["p"], wbg_s, b.ang_is, b.ang_js, g_agg, gp.w2, gp.ln, g_pre,
                                    gw_i, gw_j, g_p, None)
                    rec["bond"][t] = dict(g_eout=g_e.clone(), g_agg=g_agg, g_p=g_p)
                elif G is None:
                    K.bond_conv_bwd(sv["pre"], sv["p"], wbg_s, b.ang_is, b.ang_js, g_agg, gp.w2, gp.ln, g_pre,
                                    gw_i, gw_j)
                else:
                    g_p, g_ln = self._new(b, A, 128), ln_acc()
                    K.bond_conv_bwd(sv["pre"], sv["p"], wbg_s, b.ang_is, b.ang_js, g_agg, gp.w2, gp.ln, g_pre,
                                    gw_i, gw_j, g_p, g_ln)
                    w2_grads(f"bond.{t}", sv["pre"], g_p, g_ln)
                    G[f"bond.{t}.wo_t"] = self._wgrad(b, sv["agg"], g_e, 64, g_rows=sid)
                    if gp.extra["bo"] is not None:
                        G[f"bond.{t}.bo"] = self._colsum(b, g_e)  # identity compaction when a bias exists
                g_a = acc(g_a, g_pre, gp.extra["w1a_b"])
                g_x, g_e = angle_scatter(g_pre, g_x, g_e, gp.extra, f"bond.{t}", sv)
                K.segment_sum(gw_i, None, b.ptr_is, 1, g_wbg)
                K.segment_sum(gw_j, b.perm_js, b.ptr_js, 1, g_wbg)
            g_x, g_e = atom_conv_bwd(t, g_x, g_e)

        # ---- geometry reverse: dE/dr per directed edge -> force, virial ------------
        g_dist = self._new(b, Eu)
        g_wbg_full = self._zeros(b, Eu, 64)
        if has_ang:
            K.scatter_rows(g_wbg, sid, g_wbg_full)
        if G is not None:
            # embeddings, basis weights and the learnable basis frequencies (basis.py:23-27, 74-80)
            R, NA = pw.freq_ag.shape[0], pw.wang.shape[1]
            order = torch.argsort(b.z.long(), stable=True).int()
            zptr = torch.zeros(95, dtype=torch.int32, device=b.z.device)
            zptr[1:] = torch.cumsum(torch.bincount(b.z.long() - 1, minlength=94), 0)
            G["emb"] = self._new(b, 94, 64)
            K.segment_sum(g_x, order, zptr, 0, G["emb"])
            G["w3t"] = torch.stack([self._wgrad(b, tr["bb"], g_e, 64)[:R], self._wgrad(b, tr["bb"], g_wag, 64)[:R],
                                    self._wgrad(b, tr["bb"], g_wbg_full, 64)[32 : 32 + R]])
            g_freq = self._zeros(b, 2, R, dtype=torch.float64)
            K.bond_basis_bwd(dist, b.u2d, pw.freq_ag, pw.freq_bg, hp.atom_graph_cutoff, hp.bond_graph_cutoff,
                             hp.cutoff_coeff, pw.w3, g_e, g_wag, g_wbg_full, g_dist, g_freq)
            G["freq_ag"], G["freq_bg"] = g_freq[0].to(g_e.dtype), g_freq[1].to(g_e.dtype)
            if g_a is not None:  # None with one block: the angle features feed nothing
                G["wang_t"] = self._wgrad(b, tr["fb"], g_a, 64)[:NA]
                g_fa = self._zeros(b, pw.freq_ang.shape[0], dtype=torch.float64)
                K.angle_basis_bwd(rhat, b.ang_di, b.ang_dj, pw.freq_ang, pw.wang, g_a, None, g_fa)
                G["freq_ang"] = g_fa.to(g_e.dtype)
            return
        if rec is not None:
            rec.update(g_e0=g_e, g_wag=g_wag, g_wbg_full=g_wbg_full, g_a0=g_a)
        K.bond_basis_bwd(dist, b.u2d, pw.freq_ag, pw.freq_bg, hp.atom_graph_cutoff, hp.bond_graph_cutoff,
                         hp.cutoff_coeff, pw.w3, g_e, g_wag, g_wbg_full, g_dist)
        g_rhat = self._zeros(b, Ed, 3, dtype=torch.float64)
        if g_a is not None:  # with one block no BondConv reverse ran: dE/d(angle basis) = 0, g_rhat stays zero
            K.angle_basis_bwd(rhat, b.ang_di, b.ang_dj, pw.freq_ang, pw.wang, g_a, g_rhat)
        if rec is not None:  # adjoints of the tangent inputs ddist, drhat (Hessian-vector products)
            rec.update(g_dist=g_dist, g_rhat=g_rhat)
        force = self._zeros(b, N, 3, dtype=torch.float64)
        virial = self._zeros(b, B, 9, dtype=torch.float64)
        K.force_virial(rvec, dist, rhat, g_rhat, g_dist, b.d2u, b.u2d, b.center, b.nbr, b.owner, force, virial)
        out.force, out.virial = force, virial
