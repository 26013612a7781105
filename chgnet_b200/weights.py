"""Pack a reference ``state_dict`` into the layouts the kernels read.

The ``nn.Module`` parameters (reference names, SURVEY.md §8 a-0) stay the single
source of truth; this module only produces re-arranged *views/copies* of them
(transposes, concatenations, the split of every GatedMLP first layer into its
per-atom / per-bond / per-angle column blocks).  Call again after a parameter
update.

First-layer split (the algebraic core of the H100 design, DESIGN.md §3):
``W1 [x_c | e_u | x_n] = W1[:, 0:64] x_c + W1[:, 64:128] e_u + W1[:, 128:192] x_n``
so the 192->128 (AtomConv, reference layers.py:113-117) and 256->128 (BondConv /
AngleUpdate, layers.py:238-244, 348-355) products are computed once per ATOM and
once per BOND instead of once per edge / angle.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import torch
from torch import Tensor


@dataclass
class HyperParams:
    num_radial: int = 31
    num_angular: int = 31
    n_conv: int = 4
    atom_graph_cutoff: float = 6.0
    bond_graph_cutoff: float = 3.0
    cutoff_coeff: int = 8
    use_ln: bool = True
    readout_ln: bool = True
    is_intensive: bool = True
    n_readout_hidden: int = 3


@dataclass
class GatedPack:
    """One GatedMLP, split by input block."""

    w2t: Tensor | None = None  # [64][128] block halves (core|gate), k-major
    w2: Tensor | None = None  # [128][64] PyTorch layout stacked (core;gate)
    b2: Tensor | None = None  # [128]
    ln: Tensor | None = None  # [4][64]: g1, b1, g2, b2
    extra: dict = field(default_factory=dict)


@dataclass
class PackedWeights:
    hp: HyperParams
    emb: Tensor
    freq_ag: Tensor
    freq_bg: Tensor
    freq_ang: Tensor
    w3t: Tensor  # [3][R][64]
    w3: Tensor  # [3][64][R]
    wang_t: Tensor  # [NA][64]
    wang: Tensor  # [64][NA]
    atom: list[GatedPack]
    bond: list[GatedPack]
    angle: list[GatedPack]
    readout_ln: Tensor | None
    mlp_wt: Tensor
    mlp_w: Tensor
    mlp_b: Tensor
    w_last: Tensor
    b_last: float
    w_mag: Tensor
    b_mag: float
    atom_ref: Tensor


def _cat_t(*blocks: Tensor) -> Tensor:
    """blocks are [out][in] slices; returns k-major [in][sum(out)] contiguous."""
    return torch.cat([b.T for b in blocks], dim=1).contiguous()


def _ln_pack(sd: dict, prefix: str) -> Tensor | None:
    if f"{prefix}.bn1.weight" not in sd:
        return None
    return torch.stack(
        [sd[f"{prefix}.bn1.weight"], sd[f"{prefix}.bn1.bias"], sd[f"{prefix}.bn2.weight"], sd[f"{prefix}.bn2.bias"]]
    ).contiguous()


MAX_CONV = 8  # CHG_MAX_CONV (include/chgnet_b200.h)
MAX_READOUT_HIDDEN = 4  # MAX_HIDDEN of csrc/readout.cu and csrc/train.cu


def check_architecture(num_radial: int, num_angular: int, n_conv: int, readout_widths: list[int]) -> None:
    """Raise for a shape the kernels cannot run.  The radial basis is one lane of a warp per function (1..32), the
    Fourier basis one lane per function with the constant term (odd, 1..31), the native schedule holds up to
    ``MAX_CONV`` blocks, and the readout kernels take 1..``MAX_READOUT_HIDDEN`` hidden layers of width 64."""
    if not 1 <= num_radial <= 32:
        raise ValueError(f"num_radial={num_radial} is outside 1..32 (the radial basis is one warp lane per function)")
    if not 1 <= num_angular <= 31 or num_angular % 2 != 1:
        raise ValueError(f"num_angular={num_angular} must be odd and within 1..31 (one warp lane per Fourier function)")
    if not 1 <= n_conv <= MAX_CONV:
        raise ValueError(f"n_conv={n_conv} is outside 1..{MAX_CONV}")
    if not 1 <= len(readout_widths) <= MAX_READOUT_HIDDEN:
        raise NotImplementedError(f"mlp_hidden_dims={list(readout_widths)}: the readout kernels take 1 to "
                                  f"{MAX_READOUT_HIDDEN} hidden layers")
    if any(int(w) != 64 for w in readout_widths):
        raise NotImplementedError(f"mlp_hidden_dims={list(readout_widths)}: every readout hidden layer must be 64 wide")


def readout_layer_indices(sd: dict) -> tuple[list[int], int]:
    """(hidden Linear indices, last Linear index) of the readout MLP ``mlp.layers.*``, found as the reference's forward
    walks it (functions.py:81-92): hidden Linears at 0, 2, 4 ... while the layer exists and does not map to one output."""
    hidden, idx = [], 0
    while f"mlp.layers.{idx}.weight" in sd and sd[f"mlp.layers.{idx}.weight"].shape[0] != 1:
        hidden.append(idx)
        idx += 2
    last = max(int(k.split(".")[2]) for k in sd if k.startswith("mlp.layers.") and k.endswith(".weight"))
    return hidden, last


def infer_hyper_params(sd: dict, model_args: dict | None = None) -> HyperParams:
    a = model_args or {}
    hp = HyperParams()
    hp.num_radial = sd["bond_embedding.weight"].shape[1]
    hp.num_angular = sd["angle_embedding.weight"].shape[1]
    hp.n_conv = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("atom_conv_layers."))
    hp.atom_graph_cutoff = float(a.get("atom_graph_cutoff", 6.0))
    hp.bond_graph_cutoff = float(a.get("bond_graph_cutoff", 3.0))
    hp.cutoff_coeff = int(a.get("cutoff_coeff", 8))
    hp.use_ln = "atom_conv_layers.0.twoBody_atom.bn1.weight" in sd
    hp.readout_ln = "readout_norm.weight" in sd
    hp.is_intensive = bool(a.get("is_intensive", True))
    hidden, _ = readout_layer_indices(sd)
    check_architecture(hp.num_radial, hp.num_angular, hp.n_conv, [sd[f"mlp.layers.{i}.weight"].shape[0] for i in hidden])
    hp.n_readout_hidden = len(hidden)
    return hp


def pack_weights(state_dict: dict, model_args: dict | None = None, device=None, dtype=torch.float32) -> PackedWeights:
    sd = {k: v.detach().to(device=device, dtype=dtype) for k, v in state_dict.items()}
    hp = infer_hyper_params(sd, model_args)
    for name, dim in (("atom_embedding.embedding.weight", 1), ("bond_embedding.weight", 0), ("angle_embedding.weight", 0)):
        if sd[name].shape[dim] != 64:
            raise NotImplementedError("chgnet_b200 kernels are built for atom/bond/angle_fea_dim == 64")
    if any("bn1.running_mean" in k for k in sd):
        raise NotImplementedError("gMLP_norm='batch' is not supported by the CUDA path")

    def gated(prefix: str, first: str, second: str | None) -> tuple[Tensor, Tensor, Tensor, GatedPack]:
        w1c, w1g = sd[f"{prefix}.mlp_core.{first}.weight"], sd[f"{prefix}.mlp_gate.{first}.weight"]
        b1 = torch.cat([sd[f"{prefix}.mlp_core.{first}.bias"], sd[f"{prefix}.mlp_gate.{first}.bias"]]).contiguous()
        gp = GatedPack(ln=_ln_pack(sd, prefix))
        if second is not None:
            w2c, w2g = sd[f"{prefix}.mlp_core.{second}.weight"], sd[f"{prefix}.mlp_gate.{second}.weight"]
            if w2c.shape != (64, 64):
                raise NotImplementedError("GatedMLP hidden_dim must be 64")
            gp.w2t = _cat_t(w2c, w2g)
            gp.w2 = torch.cat([w2c, w2g], dim=0).contiguous()
            gp.b2 = torch.cat([sd[f"{prefix}.mlp_core.{second}.bias"], sd[f"{prefix}.mlp_gate.{second}.bias"]]).contiguous()
        return w1c, w1g, b1, gp

    atom, bond, angle = [], [], []
    for t in range(hp.n_conv):
        w1c, w1g, b1, gp = gated(f"atom_conv_layers.{t}.twoBody_atom", "layers.0", "layers.3")
        if w1c.shape != (64, 192):
            raise NotImplementedError("AtomConv GatedMLP must be 192 -> 64 -> 64")
        cen, bnd, nbr = slice(0, 64), slice(64, 128), slice(128, 192)
        wo = sd[f"atom_conv_layers.{t}.mlp_out.layers.1.weight"]
        gp.extra = dict(
            wcn_t=_cat_t(w1c[:, cen], w1g[:, cen], w1c[:, nbr], w1g[:, nbr]),  # [64][256]
            we_t=_cat_t(w1c[:, bnd], w1g[:, bnd]),  # [64][128]
            b1=b1,
            wcn_b=torch.cat([w1c[:, cen], w1g[:, cen], w1c[:, nbr], w1g[:, nbr]], dim=0).contiguous(),  # [256][64]
            we_b=torch.cat([w1c[:, bnd], w1g[:, bnd]], dim=0).contiguous(),  # [128][64]
            wo_t=wo.T.contiguous(),
            wo=wo.contiguous(),
            bo=sd.get(f"atom_conv_layers.{t}.mlp_out.layers.1.bias"),
        )
        atom.append(gp)
    bi, bj, an, xc = slice(0, 64), slice(64, 128), slice(128, 192), slice(192, 256)
    for t in range(hp.n_conv - 1):
        if f"bond_conv_layers.{t}.twoBody_bond.mlp_core.layers.0.weight" not in sd:
            raise NotImplementedError("update_bond=False models are not supported")
        w1c, w1g, b1, gp = gated(f"bond_conv_layers.{t}.twoBody_bond", "layers.0", "layers.3")
        wo = sd[f"bond_conv_layers.{t}.mlp_out.layers.1.weight"]
        gp.extra = dict(
            wij_t=_cat_t(w1c[:, bi], w1g[:, bi], w1c[:, bj], w1g[:, bj]),  # [64][256]
            bij=torch.cat([b1, torch.zeros_like(b1)]).contiguous(),  # bias rides on the i half
            wx_t=_cat_t(w1c[:, xc], w1g[:, xc]),
            w1a_t=_cat_t(w1c[:, an], w1g[:, an]),
            wij_b=torch.cat([w1c[:, bi], w1g[:, bi], w1c[:, bj], w1g[:, bj]], dim=0).contiguous(),
            wx_b=torch.cat([w1c[:, xc], w1g[:, xc]], dim=0).contiguous(),
            w1a_b=torch.cat([w1c[:, an], w1g[:, an]], dim=0).contiguous(),
            wo_t=wo.T.contiguous(),
            wo=wo.contiguous(),
            bo=sd.get(f"bond_conv_layers.{t}.mlp_out.layers.1.bias"),
        )
        bond.append(gp)
        if f"angle_layers.{t}.twoBody_bond.mlp_core.layers.1.weight" not in sd:
            raise NotImplementedError("update_angle=False / hidden angle layers are not supported")
        w1c, w1g, b1, gp = gated(f"angle_layers.{t}.twoBody_bond", "layers.1", None)
        gp.extra = dict(
            wij_t=_cat_t(w1c[:, bi], w1g[:, bi], w1c[:, bj], w1g[:, bj]),
            bij=torch.cat([b1, torch.zeros_like(b1)]).contiguous(),
            wx_t=_cat_t(w1c[:, xc], w1g[:, xc]),
            w1a_t=_cat_t(w1c[:, an], w1g[:, an]),
            wij_b=torch.cat([w1c[:, bi], w1g[:, bi], w1c[:, bj], w1g[:, bj]], dim=0).contiguous(),
            wx_b=torch.cat([w1c[:, xc], w1g[:, xc]], dim=0).contiguous(),
            w1a_b=torch.cat([w1c[:, an], w1g[:, an]], dim=0).contiguous(),
        )
        angle.append(gp)

    hidden_idx, last_idx = readout_layer_indices(sd)
    mlp_w = torch.stack([sd[f"mlp.layers.{i}.weight"] for i in hidden_idx]).contiguous()
    return PackedWeights(
        hp=hp,
        emb=sd["atom_embedding.embedding.weight"].contiguous(),
        freq_ag=sd["bond_basis_expansion.rbf_expansion_ag.frequencies"].contiguous(),
        freq_bg=sd["bond_basis_expansion.rbf_expansion_bg.frequencies"].contiguous(),
        freq_ang=sd["angle_basis_expansion.fourier_expansion.frequencies"].contiguous(),
        w3t=torch.stack(
            [sd["bond_embedding.weight"].T, sd["bond_weights_ag.weight"].T, sd["bond_weights_bg.weight"].T]
        ).contiguous(),
        w3=torch.stack(
            [sd["bond_embedding.weight"], sd["bond_weights_ag.weight"], sd["bond_weights_bg.weight"]]
        ).contiguous(),
        wang_t=sd["angle_embedding.weight"].T.contiguous(),
        wang=sd["angle_embedding.weight"].contiguous(),
        atom=atom,
        bond=bond,
        angle=angle,
        readout_ln=(
            torch.stack([sd["readout_norm.weight"], sd["readout_norm.bias"]]).contiguous() if hp.readout_ln else None
        ),
        mlp_wt=mlp_w.transpose(1, 2).contiguous(),
        mlp_w=mlp_w,
        mlp_b=torch.stack([sd[f"mlp.layers.{i}.bias"] for i in hidden_idx]).contiguous(),
        w_last=sd[f"mlp.layers.{last_idx}.weight"].reshape(-1).contiguous(),
        b_last=float(sd[f"mlp.layers.{last_idx}.bias"].reshape(-1)[0]),
        w_mag=sd["site_wise.weight"].reshape(-1).contiguous(),
        b_mag=float(sd["site_wise.bias"].reshape(-1)[0]),
        atom_ref=(
            sd["composition_model.fc.weight"].reshape(-1).contiguous()
            if "composition_model.fc.weight" in sd
            else torch.zeros(94, device=device, dtype=dtype)
        ),
    )


def unpack_grads(G: dict, state_dict: dict) -> dict[str, Tensor]:
    """Inverse of :func:`pack_weights` for GRADIENTS: the packed-layout gradients produced by
    ``Engine.param_grads`` -> one tensor per ``state_dict`` name (same shapes).

    Parameters the loss cannot reach get zeros (``angle_layers.{n_conv-2}`` is dead compute in
    the reference, model.py:470-496; ``composition_model`` is frozen, composition_model.py:127-131).
    """
    sd = state_dict
    out: dict[str, Tensor] = {}
    any_g = G["emb"]

    def put(name: str, val) -> None:
        if name in sd:
            out[name] = torch.as_tensor(val, dtype=any_g.dtype, device=any_g.device).reshape(sd[name].shape)

    def gated(prefix: str, key: str, first: str, second: str | None, blocks: list[tuple[str, int, int]]) -> None:
        """blocks: (packed key, core column offset, gate column offset) per 64-wide input block, in
        the reference's concatenation order."""
        if f"{key}.{blocks[0][0]}" not in G:
            return
        put(f"{prefix}.mlp_core.{first}.weight", torch.cat([G[f"{key}.{k}"][:, c : c + 64].T for k, c, _ in blocks], dim=1))
        put(f"{prefix}.mlp_gate.{first}.weight", torch.cat([G[f"{key}.{k}"][:, g : g + 64].T for k, _, g in blocks], dim=1))
        put(f"{prefix}.mlp_core.{first}.bias", G[f"{key}.b1"][:64])
        put(f"{prefix}.mlp_gate.{first}.bias", G[f"{key}.b1"][64:])
        if second is not None:
            put(f"{prefix}.mlp_core.{second}.weight", G[f"{key}.w2t"][:, :64].T)
            put(f"{prefix}.mlp_gate.{second}.weight", G[f"{key}.w2t"][:, 64:].T)
            put(f"{prefix}.mlp_core.{second}.bias", G[f"{key}.b2"][:64])
            put(f"{prefix}.mlp_gate.{second}.bias", G[f"{key}.b2"][64:])
        if f"{key}.ln" in G:
            for i, nm in enumerate(("bn1.weight", "bn1.bias", "bn2.weight", "bn2.bias")):
                put(f"{prefix}.{nm}", G[f"{key}.ln"][i])

    n_conv = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("atom_conv_layers."))
    for t in range(n_conv):
        gated(f"atom_conv_layers.{t}.twoBody_atom", f"atom.{t}", "layers.0", "layers.3",
              [("wcn_t", 0, 64), ("we_t", 0, 64), ("wcn_t", 128, 192)])
        if f"atom.{t}.wo_t" in G:
            put(f"atom_conv_layers.{t}.mlp_out.layers.1.weight", G[f"atom.{t}.wo_t"].T)
            if f"atom.{t}.bo" in G:
                put(f"atom_conv_layers.{t}.mlp_out.layers.1.bias", G[f"atom.{t}.bo"])
    ij_a_x = [("wij_t", 0, 64), ("wij_t", 128, 192), ("w1a_t", 0, 64), ("wx_t", 0, 64)]
    for t in range(n_conv - 1):
        gated(f"bond_conv_layers.{t}.twoBody_bond", f"bond.{t}", "layers.0", "layers.3", ij_a_x)
        if f"bond.{t}.wo_t" in G:
            put(f"bond_conv_layers.{t}.mlp_out.layers.1.weight", G[f"bond.{t}.wo_t"].T)
            if f"bond.{t}.bo" in G:
                put(f"bond_conv_layers.{t}.mlp_out.layers.1.bias", G[f"bond.{t}.bo"])
        gated(f"angle_layers.{t}.twoBody_bond", f"angle.{t}", "layers.1", None, ij_a_x)

    put("atom_embedding.embedding.weight", G["emb"])
    put("bond_embedding.weight", G["w3t"][0].T)
    put("bond_weights_ag.weight", G["w3t"][1].T)
    put("bond_weights_bg.weight", G["w3t"][2].T)
    put("bond_basis_expansion.rbf_expansion_ag.frequencies", G["freq_ag"])
    put("bond_basis_expansion.rbf_expansion_bg.frequencies", G["freq_bg"])
    if "wang_t" in G:
        put("angle_embedding.weight", G["wang_t"].T)
        put("angle_basis_expansion.fourier_expansion.frequencies", G["freq_ang"])
    if "readout_ln" in G:
        put("readout_norm.weight", G["readout_ln"][0])
        put("readout_norm.bias", G["readout_ln"][1])
    hidden_idx, last_idx = readout_layer_indices(sd)
    for l, i in enumerate(hidden_idx):
        put(f"mlp.layers.{i}.weight", G["mlp_wt"][l].T)
        put(f"mlp.layers.{i}.bias", G["mlp_b"][l])
    put(f"mlp.layers.{last_idx}.weight", G["w_last"])
    put(f"mlp.layers.{last_idx}.bias", G["b_last"])
    if "w_mag" in G:
        put("site_wise.weight", G["w_mag"])
        put("site_wise.bias", G["b_mag"])
    for name, v in sd.items():
        if name not in out and torch.is_floating_point(torch.as_tensor(v)):
            out[name] = torch.zeros(tuple(v.shape), dtype=any_g.dtype, device=any_g.device)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Index maps: pack_weights / unpack_grads are pure re-arrangements (slices, transposes, concatenations), so running them
# ONCE on tensors that hold positions instead of values yields gather maps; afterwards the packed weights are refreshed
# from the flat parameter buffer, and the packed gradients are flattened, with one gather each (no per-tensor Python).
# ---------------------------------------------------------------------------------------------------------------------
def packed_tensors(pw: PackedWeights) -> list[tuple[object, str | tuple]]:
    """(owner, key) of every tensor of a PackedWeights in a fixed order; owner is the dataclass (attribute key) or an
    ``extra`` dict (item key)."""
    out: list[tuple[object, str | tuple]] = []
    for name in ("emb", "freq_ag", "freq_bg", "freq_ang", "w3t", "w3", "wang_t", "wang", "readout_ln", "mlp_wt", "mlp_w", "mlp_b",
                 "w_last", "w_mag", "atom_ref"):
        if getattr(pw, name) is not None:
            out.append((pw, name))
    for packs in (pw.atom, pw.bond, pw.angle):
        for gp in packs:
            for name in ("w2t", "w2", "b2", "ln"):
                if getattr(gp, name) is not None:
                    out.append((gp, name))
            for k in sorted(gp.extra):
                if gp.extra[k] is not None:
                    out.append((gp.extra, (k,)))
    return out


def _get(owner, key):
    return owner[key[0]] if isinstance(key, tuple) else getattr(owner, key)


def _set(owner, key, val) -> None:
    if isinstance(key, tuple):
        owner[key[0]] = val
    else:
        setattr(owner, key, val)


class RepackMap:
    """Refresh ``pw`` in place from the flat trainable-parameter buffer: ``pbuf[pos] = flat[src]`` (two launches).

    ``offsets`` / ``names``: where every trainable parameter sits in ``flat`` (chgnet_b200.trainer.Trainer)."""

    def __init__(self, pw: PackedWeights, state_dict: dict, model_args: dict | None, names, offsets, flat: Tensor) -> None:
        dev = flat.device
        where = dict(zip(names, offsets))
        sd_idx = {}
        for k, v in state_dict.items():
            v = torch.as_tensor(v)
            if not torch.is_floating_point(v):
                continue
            if k in where:
                sd_idx[k] = (where[k] + 1 + torch.arange(v.numel(), dtype=torch.float64, device=dev)).reshape(v.shape)
            else:  # frozen parameter / buffer: position 0 = "keep the packed value"
                sd_idx[k] = torch.zeros(v.shape, dtype=torch.float64, device=dev)
        pw_idx = pack_weights(sd_idx, model_args, device=dev, dtype=torch.float64)
        real, idx = packed_tensors(pw), packed_tensors(pw_idx)
        assert [k for _, k in real] == [k for _, k in idx]
        sizes = [(_get(o, k).numel() + 15) // 16 * 16 for o, k in real]  # 64-byte aligned pieces
        self.pbuf = torch.zeros(sum(sizes), dtype=flat.dtype, device=dev)
        src = torch.zeros(sum(sizes), dtype=torch.int64, device=dev)
        off = 0
        for (o, k), (oi, ki), sz in zip(real, idx, sizes):
            t = _get(o, k)
            view = self.pbuf[off : off + t.numel()].view(t.shape)
            view.copy_(t)
            _set(o, k, view)  # the engine now reads the shared buffer
            src[off : off + t.numel()] = _get(oi, ki).reshape(-1).long()
            off += sz
        self.pos = torch.nonzero(src > 0).view(-1)
        self.src = (src[self.pos] - 1).contiguous()
        self.scalars = torch.tensor([where.get(n, -1) for n in self._scalar_names(state_dict)], dtype=torch.int64, device=dev)
        self.pw = pw

    @staticmethod
    def _scalar_names(sd) -> tuple[str, str]:
        last = max(int(k.split(".")[2]) for k in sd if k.startswith("mlp.layers.") and k.endswith(".weight"))
        return (f"mlp.layers.{last}.bias", "site_wise.bias")

    def refresh(self, flat: Tensor) -> None:
        self.pbuf.index_copy_(0, self.pos, flat.index_select(0, self.src))
        if int(self.scalars.min()) >= 0:  # the two biases the kernels take by value
            b_last, b_mag = flat.index_select(0, self.scalars).tolist()
            self.pw.b_last, self.pw.b_mag = float(b_last), float(b_mag)


class GradFlattenMap:
    """``flat_grad = cat(0, G.values())[inv]``: the packed-layout gradients of ``Engine.param_grads`` -> the flat buffer in
    the Trainer's layout (what ``unpack_grads`` + per-parameter copies did with ~300 small launches)."""

    def __init__(self, G: dict, state_dict: dict, names, offsets, sizes, n_flat: int) -> None:
        dev = G["emb"].device
        self.signature = tuple((k, tuple(torch.as_tensor(v).shape)) for k, v in G.items())
        g_idx, off = {}, 1  # position 0 of the concatenation is a zero
        for k, v in G.items():
            v = torch.as_tensor(v)
            g_idx[k] = (off + torch.arange(v.numel(), dtype=torch.float64, device=dev)).reshape(v.shape)
            off += v.numel()
        by_name = unpack_grads(g_idx, state_dict)
        inv = torch.zeros(n_flat, dtype=torch.int64, device=dev)
        for n, o, sz in zip(names, offsets, sizes):
            inv[o : o + sz] = by_name[n].reshape(-1).long()
        self.inv = inv
        self.zero = torch.zeros(1, dtype=torch.float32, device=dev)

    def matches(self, G: dict) -> bool:
        return self.signature == tuple((k, tuple(torch.as_tensor(v).shape)) for k, v in G.items())

    def flatten(self, G: dict, out: Tensor) -> Tensor:
        cat = torch.cat([self.zero] + [torch.as_tensor(v, dtype=torch.float32, device=out.device).reshape(-1) for v in G.values()])
        torch.index_select(cat, 0, self.inv, out=out)
        return out

