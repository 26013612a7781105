"""-m gpu: the four three-phonon kernels against their fp64 specifications away from the cubic meshes, single
temperature tile and 24 / 93 band counts of the other device tests.

* ``chg_phonon_interaction``, ``chg_imag_self_energy``, ``chg_collision_rows`` and ``chg_self_energy_spectrum``
  against ``ThreePhononSpecKernels``, ``LbteSpecKernels`` and ``SpectralFunctionSpecKernels`` (run with torch on the
  same device) over a table of cases: non-cubic meshes (one with an axis of length 1), every tetrahedron diagonal and
  a sheared lattice's own choice, 3, 24, 33 and 96 bands, a non-diagonal supercell, 9 and 17 temperatures (unsorted,
  repeated, 0 K in a later tile), targets at 0, N - 1 and inside, q1 lists split off the tile sizes, single and
  permuted, frequencies on a 0.25 THz grid (ties everywhere), and 1, 32 and 33 spectrum points; two calls bitwise
  equal;
* the contracts of the kernels: the write footprint of ``chg_collision_rows``, the accumulation of
  ``chg_imag_self_energy`` and ``chg_self_energy_spectrum``, and the argument limits;
* ``chg_tetrahedron_dos`` on a non-cubic mesh, and ``Phonons.dos`` there against the specification path;
* on the device fc3 of LiMnO2 2x2x2 on a non-cubic mesh at 9 temperatures, ``linewidths``, ``thermal_conductivity``,
  ``thermal_conductivity_lbte`` and ``spectral_function`` against the specification path, and with the q1 chunks and
  the temperature groups split."""
import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200._lib import ChgnetB200Error
from chgnet_b200.phonons import THERMAL_CUTOFF_THZ, Phonons, tetrahedra
from lbte_kernels import LbteSpecKernels
from oracle.phonons import PhononSpecKernels
from spectral_function_kernels import SpectralFunctionSpecKernels
from test_spectral_function_gpu import _random_p
from test_three_phonon_gpu import _random_case
from three_phonon_kernels import ThreePhononSpecKernels

pytestmark = pytest.mark.gpu
CUT = THERMAL_CUTOFF_THZ

NONDIAGONAL = [[0, 1, 1], [1, 0, 1], [1, 1, 0]]
# on the (4, 3, 5) mesh the shortest body diagonal of this lattice's mesh cell is diagonal 1 (0.084 1/A, against 0.092,
# 0.121 and 0.134)
SHEARED = np.array([[4.0, 0.0, 0.0], [-2.0, 4.5, 0.0], [0.0, 1.0, 5.0]])
T9 = [0.0, 10.0, 50.0, 100.0, 300.0, 500.0, 1000.0, 2000.0, 1e4]
# unsorted, 300 K twice, and 0 K last: the one-temperature tail tile of chg_imag_self_energy (tiles of 8) and of
# chg_collision_rows and chg_self_energy_spectrum (tiles of 4)
T17 = [300.0, 1000.0, 50.0, 2000.0, 10.0, 500.0, 300.0, 5000.0, 100.0, 20.0, 700.0, 1e4, 150.0, 3000.0, 30.0, 250.0,
       0.0]


def _case(n_prim, cells, mesh, seed, tets=None, quantised=False):
    """``_random_case`` with the tetrahedra of ``tets`` (None: its own; 0 - 3: that diagonal; "sheared": the choice
    for ``SHEARED``) and, if ``quantised``, its frequencies rounded to 0.25 THz with band 1 set to the cutoff, 0 and
    -0.25 in turn, so that corner sums land exactly on band frequencies and on 0.25 THz points."""
    args, nu, e, t = _random_case(n_prim, cells, mesh, seed)
    if tets == "sheared":
        t = torch.as_tensor(tetrahedra(mesh, SHEARED)).cuda()
    elif tets is not None:
        t = torch.as_tensor(tetrahedra(mesh, np.eye(3), diagonal=tets)).cuda()
    if quantised:
        nu = torch.round(nu * 4) / 4
        nu[0::3, 1], nu[1::3, 1], nu[2::3, 1] = CUT, 0.0, -0.25
        nu = torch.sort(nu, dim=1)[0].contiguous()
    return args, nu, e, t


def _points(n_freq, nu, quantised):
    """Ascending spectrum points: one inside the bands, or 0, one below the cutoff and the cutoff itself then a
    uniform grid up to 2 max(nu) (quantised: 0 and multiples of 0.25 THz)."""
    top = 2 * float(nu.max())
    if n_freq == 1:
        return torch.tensor([0.6 * top], dtype=torch.float64, device="cuda")
    if quantised:
        step = 0.25 * np.ceil(top / (0.25 * (n_freq - 1)))
        return torch.arange(n_freq, dtype=torch.float64, device="cuda") * step
    rest = torch.linspace(CUT, top, n_freq - 2, dtype=torch.float64, device="cuda")
    return torch.cat([torch.tensor([0.0, 5e-4], dtype=torch.float64, device="cuda"), rest])


def _q1_list(kind, n_mesh, nb, seed):
    """(q1 int32, call boundaries): the whole mesh in three calls cut at 7 and 2N/3 + 1 (off every tile size), one
    q1, or a permuted subset (4 q1 at 96 bands, else N/2 + 1) in one call."""
    if kind == "split":
        q1 = torch.arange(n_mesh, dtype=torch.int32, device="cuda")
        return q1, sorted({0, 7, 2 * n_mesh // 3 + 1, n_mesh})
    if kind == "one":
        return torch.tensor([n_mesh - 2], dtype=torch.int32, device="cuda"), [0, 1]
    g = torch.Generator(device="cuda").manual_seed(seed)
    q1 = torch.randperm(n_mesh, generator=g, device="cuda")[: 4 if nb > 64 else n_mesh // 2 + 1].to(torch.int32)
    return (q1.flip(0) if bool((q1[1:] > q1[:-1]).all()) else q1), [0, len(q1)]


# n_prim, supercell, mesh, target (-1: N - 1), temperatures, q1 list, tetrahedra, quantised, spectrum points
CASES = {
    "m435-b24-split-t28-T9-f33": (8, (2, 2, 2), (4, 3, 5), 28, T9, "split", None, False, 33),
    "m614-b24-perm-t0-T17-f32": (8, (2, 2, 2), (6, 1, 4), 0, T17, "perm", None, False, 32),
    "m352-b24-one-tlast-T9-f33": (8, (2, 2, 2), (3, 5, 2), -1, T9, "one", None, False, 33),
    "m614-b24-perm-t11-T9-f1": (8, (2, 2, 2), (6, 1, 4), 11, T9, "perm", None, False, 1),
    "m435-b24-diag0": (8, (2, 2, 2), (4, 3, 5), 28, T9, "split", 0, False, 33),
    "m435-b24-diag1": (8, (2, 2, 2), (4, 3, 5), 28, T9, "split", 1, False, 33),
    "m435-b24-diag2": (8, (2, 2, 2), (4, 3, 5), 28, T9, "split", 2, False, 33),
    "m435-b24-diag3": (8, (2, 2, 2), (4, 3, 5), 28, T9, "split", 3, False, 33),
    "m435-b24-sheared-tlast-T17-f32": (8, (2, 2, 2), (4, 3, 5), -1, T17, "split", "sheared", False, 32),
    "m352-b3-split-t0-T17-f33": (1, (2, 2, 2), (3, 5, 2), 0, T17, "split", None, False, 33),
    "m435-b33-perm-t28-T9-f33": (11, (2, 1, 1), (4, 3, 5), 28, T9, "perm", None, False, 33),
    "m352-b96-perm-t16-T9-f33": (32, (2, 1, 1), (3, 5, 2), 16, T9, "perm", None, False, 33),
    "m614-b12-nondiagonal-tlast-T17-f32": (4, NONDIAGONAL, (6, 1, 4), -1, T17, "split", None, False, 32),
    "m435-b24-quantised-t28-T9-f33": (8, (2, 2, 2), (4, 3, 5), 28, T9, "split", None, True, 33),
}


@pytest.mark.parametrize("case", list(CASES))
def test_kernels_match_spec_on_shapes(case):
    from chgnet_b200._lib import CudaKernels

    n_prim, cells, mesh, target, temps, q1_kind, tets_kind, quantised, n_freq = CASES[case]
    seed = list(CASES).index(case) + 100
    args, nu, e, tets = _case(n_prim, cells, mesh, seed, tets_kind, quantised)
    n_mesh, nb = int(np.prod(mesh)), 3 * n_prim
    target = n_mesh - 1 if target < 0 else target
    if tets_kind == "sheared":
        assert tetrahedra(mesh, SHEARED).tolist() == tetrahedra(mesh, np.eye(3), diagonal=1).tolist()
    if cells is NONDIAGONAL:
        counts = args[1][1:] - args[1][:-1]
        assert int(counts.max()) > 1  # pairs with several minimum images
    q1, cuts = _q1_list(q1_kind, n_mesh, nb, seed)
    t = torch.tensor(temps, dtype=torch.float64, device="cuda")
    omega = nu[target].contiguous()
    points = _points(n_freq, nu, quantised)
    kern = CudaKernels("cuda")
    spec_p, spec, spec_sf = ThreePhononSpecKernels(), LbteSpecKernels(), SpectralFunctionSpecKernels()
    calls = list(zip(cuts[:-1], cuts[1:]))

    def interaction(k):
        p = torch.empty(len(q1), nb, nb, nb, dtype=torch.float64, device="cuda")
        for s, u in calls:
            k.phonon_interaction(*args, mesh, nu, e, target, q1[s:u], CUT, p[s:u])
        return p

    def consumers(k, k_sf, p):
        gamma = torch.zeros(len(t), nb, dtype=torch.float64, device="cuda")
        rows = torch.zeros(4, len(t), nb, n_mesh, nb, dtype=torch.float64, device="cuda")
        se = torch.zeros(len(t), nb, n_freq, dtype=torch.float64, device="cuda")
        for s, u in calls:
            k.imag_self_energy(nu, mesh, tets, target, omega, q1[s:u], p[s:u], t, CUT, gamma)
            k.collision_rows(nu, mesh, tets, target, omega, q1[s:u], p[s:u], t, CUT, rows)
            k_sf.self_energy_spectrum(nu, mesh, tets, target, points, q1[s:u], p[s:u], t, CUT, se)
        return gamma, rows, se

    pk = interaction(kern)
    assert torch.equal(pk, interaction(kern))
    got = consumers(kern, kern, pk)
    for a, b in zip(got, consumers(kern, kern, pk)):
        assert torch.equal(a, b)
    # the consumers get the device P on both sides, so that each kernel is compared on its own
    want = (interaction(spec_p),) + consumers(spec, spec_sf, pk)
    errs = {}
    for name, g, w in zip(("P", "Gamma", "rows", "spectrum"), (pk,) + got, want):
        scale = float(w.abs().max())
        assert scale > 0 and bool(torch.isfinite(g).all()), name
        errs[name] = float((g - w).abs().max()) / scale
    print(f"{case}: {nb} bands on {mesh}, target {target}, {len(q1)} q1 in {len(calls)} calls, {len(temps)} "
          f"temperatures, {n_freq} points: bitwise reproducible; against the specification "
          + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert errs["P"] <= 1e-12 and errs["Gamma"] <= 1e-11 and errs["rows"] <= 5e-15 and errs["spectrum"] <= 5e-15


def test_collision_rows_write_footprint():
    from chgnet_b200._lib import CudaKernels

    mesh = (4, 3, 5)
    _, nu, _, tets = _case(8, (2, 2, 2), mesh, 7)
    n_mesh, nb = nu.shape
    nu[13] = torch.linspace(-0.5, -0.05, nb, dtype=torch.float64, device="cuda")  # every nu1 at q1 = 13 below the cutoff
    targets = (28, 41)
    temps = torch.tensor(T9, dtype=torch.float64, device="cuda")
    q1 = torch.tensor([40, 13, 2, 57, 21, 9], dtype=torch.int32, device="cuda")
    kern, spec = CudaKernels("cuda"), LbteSpecKernels()
    fill = torch.full((4, len(temps), nb, n_mesh, nb), float("nan"), dtype=torch.float64, device="cuda")
    out = fill.clone()
    others = torch.ones(n_mesh, dtype=torch.bool, device="cuda")
    others[q1.long()] = False
    for i, target in enumerate(targets):  # the second target reuses the first one's out, as _collision_passes does
        p = _random_p(nu, mesh, target, 11 + i)[q1.long()].contiguous()
        p[3] = 0.0  # q1 = 57: P all zero
        assert not bool(p[1].any())  # q1 = 13: _random_p leaves out nu1 below the cutoff
        omega = nu[target].contiguous()
        kern.collision_rows(nu, mesh, tets, target, omega, q1, p, temps, CUT, out)
        want = torch.zeros_like(out)
        spec.collision_rows(nu, mesh, tets, target, omega, q1, p, temps, CUT, want)
        cols = out[:, :, :, q1.long()]
        scale = float(want.abs().max())
        err = float((cols - want[:, :, :, q1.long()]).abs().max()) / scale
        print(f"collision rows, target {target}, 6 of {n_mesh} q1 into a NaN-filled out: columns written "
              f"{err:.2e} of max|R| against the specification; the other {int(others.sum())} columns untouched")
        assert scale > 0 and bool(torch.isfinite(cols).all()) and err <= 5e-15
        assert not bool(cols[:, :, :, 1].any()) and not bool(cols[:, :, :, 3].any())
        assert torch.equal(out[:, :, :, others].view(torch.int64), fill[:, :, :, others].view(torch.int64))


def test_gamma_outputs_accumulate():
    from chgnet_b200._lib import CudaKernels

    mesh, target = (6, 1, 4), 11
    _, nu, _, tets = _case(8, (2, 2, 2), mesh, 8)
    n_mesh, nb = nu.shape
    p = _random_p(nu, mesh, target, 12)
    q1 = torch.arange(n_mesh, dtype=torch.int32, device="cuda")
    temps = torch.tensor(T17, dtype=torch.float64, device="cuda")
    points = _points(33, nu, False)
    omega = nu[target].contiguous()
    kern = CudaKernels("cuda")
    g = torch.Generator(device="cuda").manual_seed(5)
    for name, shape, call, tol in (
            ("imag_self_energy", (len(temps), nb),
             lambda out: kern.imag_self_energy(nu, mesh, tets, target, omega, q1, p, temps, CUT, out), 1e-11),
            ("self_energy_spectrum", (len(temps), nb, len(points)),
             lambda out: kern.self_energy_spectrum(nu, mesh, tets, target, points, q1, p, temps, CUT, out), 5e-15)):
        fresh = torch.zeros(shape, dtype=torch.float64, device="cuda")
        call(fresh)
        start = (torch.rand(shape, generator=g, device="cuda", dtype=torch.float64) + 0.5) * fresh.abs().max()
        acc = start.clone()
        call(acc)
        err = float((acc - (start + fresh)).abs().max() / (start + fresh).abs().max())
        print(f"{name}: into a random nonzero output vs initial value + fresh result {err:.2e}")
        assert float(fresh.abs().max()) > 0 and err <= tol


def test_argument_limits():
    from chgnet_b200._lib import CudaKernels

    kern = CudaKernels("cuda")

    def rejected(call, match):
        before = kern.launches
        with pytest.raises(ChgnetB200Error, match=match):
            call()
        assert kern.launches == before  # nothing launched

    f64, i32 = torch.float64, torch.int32
    # collision rows: 769 bands rejected before the early return of an empty call; 768 accepted
    one = (1, 1, 1)
    tets1 = torch.as_tensor(tetrahedra(one, np.eye(3))).cuda()
    temps = torch.tensor([300.0], dtype=f64, device="cuda")
    none = torch.zeros(0, dtype=i32, device="cuda")
    for nb, ok in ((768, True), (769, False)):
        nu = torch.linspace(1.0, 20.0, nb, dtype=f64, device="cuda")[None].contiguous()
        p = torch.zeros(0, nb, nb, nb, dtype=f64, device="cuda")
        out = torch.zeros(4, 1, nb, 1, nb, dtype=f64, device="cuda")
        call = lambda: kern.collision_rows(nu, one, tets1, 0, nu[0].contiguous(), none, p, temps, CUT, out)  # noqa
        if ok:
            call()
        else:
            rejected(call, "too many bands")
    # the interaction: at most 65 535 q1 in one call (3 bands, a one-point mesh)
    args, nu, e, _ = _random_case(1, (1, 1, 1), one, 3)
    for n_q1, ok in ((65535, True), (65536, False)):
        q1 = torch.zeros(n_q1, dtype=i32, device="cuda")
        out = torch.full((n_q1, 3, 3, 3), float("nan"), dtype=f64, device="cuda")
        if ok:
            kern.phonon_interaction(*args, one, nu, e, 0, q1, CUT, out)
            assert bool(torch.isfinite(out).all()) and torch.equal(out, out[:1].expand_as(out))
        else:
            rejected(lambda: kern.phonon_interaction(*args, one, nu, e, 0, q1, CUT, out), "too many q1")
    # a target outside the mesh, for each kernel
    mesh = (2, 3, 1)
    args, nu, e, tets = _case(1, (2, 2, 2), mesh, 4)
    q1 = torch.arange(6, dtype=i32, device="cuda")
    p = torch.zeros(6, 3, 3, 3, dtype=f64, device="cuda")
    omega = nu[0].contiguous()
    for target in (-1, 6):
        for call in (lambda: kern.phonon_interaction(*args, mesh, nu, e, target, q1, CUT, p),
                     lambda: kern.imag_self_energy(nu, mesh, tets, target, omega, q1, p, temps, CUT,
                                                   torch.zeros(1, 3, dtype=f64, device="cuda")),
                     lambda: kern.collision_rows(nu, mesh, tets, target, omega, q1, p, temps, CUT,
                                                 torch.zeros(4, 1, 3, 6, 3, dtype=f64, device="cuda")),
                     lambda: kern.self_energy_spectrum(nu, mesh, tets, target, omega, q1, p, temps, CUT,
                                                       torch.zeros(1, 3, 3, dtype=f64, device="cuda"))):
            rejected(call, "target outside the mesh")
    torch.cuda.synchronize()


def test_tetrahedron_dos_non_cubic_mesh():
    from chgnet_b200._lib import CudaKernels

    rng = np.random.default_rng(37)
    mesh = (20, 12, 7)
    n_q, n_band, n_proj = int(np.prod(mesh)), 24, 7
    # values on a 1/8 THz grid: vertices tie often, and every frequency point below sits on possible vertex values
    freqs = np.sort(np.round(rng.uniform(-2.0, 20.0, size=(n_q, n_band)) * 8) / 8, axis=1)
    proj = rng.uniform(0.0, 1.0, size=(n_q, n_band, n_proj))
    omega = np.arange(-2.5, 20.5, 0.125)
    dev = torch.device("cuda")
    f, p, w = (torch.as_tensor(x).to(dev) for x in (freqs, proj, omega))
    tets = torch.as_tensor(tetrahedra(mesh, SHEARED)).to(dev)
    kern = CudaKernels(dev)

    def run(k):
        out = [torch.full((len(omega),), float("nan"), dtype=torch.float64, device=dev) for _ in range(2)]
        pd = torch.full((n_proj, len(omega)), float("nan"), dtype=torch.float64, device=dev)
        k.tetrahedron_dos(f, mesh, tets, w, out[0], out[1], p, pd)
        return out + [pd]

    got, again, want = run(kern), run(kern), run(PhononSpecKernels())
    for name, a, b, c in zip(("dos", "idos", "pdos"), got, again, want):
        scale = float(c.abs().max())
        err = float((a - c).abs().max()) / scale
        print(f"tetrahedron dos {mesh}, {n_band} bands, {len(omega)} points: {name} max|kernel - spec| / max = {err:.2e}")
        assert err <= 1e-10 and torch.equal(a, b)
    assert abs(float(got[1][-1]) - n_band) <= 1e-12 * n_band


@pytest.fixture(scope="module")
def limno2_fc3():
    model = phonon_cells.model030()
    return model.phonons(graphgen.limno2_structure(), [2, 2, 2], third_order=True)


MESH = (6, 4, 3)
Q = np.array([[0.0, 0.0, 0.0], [1 / 3, 1 / 4, 2 / 3], [0.5, 0.5, 1 / 3], [5 / 6, 0.75, 0.0]])
SF_Q = Q[1:3]


def _errs(got, want, keys):
    return {k: float(np.abs(got[k] - want[k]).max() / np.abs(want[k]).max()) for k in keys}


def _methods(ph, which=("linewidths", "rta", "lbte", "spectral")):
    out = {}
    if "linewidths" in which:
        out["linewidths"] = ph.linewidths(MESH, Q, T9)
    if "rta" in which:
        out["rta"] = ph.thermal_conductivity(MESH, T9)
    if "lbte" in which:
        out["lbte"] = ph.thermal_conductivity_lbte(MESH, T9)
    if "spectral" in which:
        out["spectral"] = ph.spectral_function(MESH, SF_Q, T9)
    return out


@pytest.fixture(scope="module")
def unsplit(limno2_fc3):
    return _methods(limno2_fc3)


def _check(got, want, label):
    """Asserts the method-level tolerances of got against want (both ``_methods`` results) for the methods in got."""
    if "linewidths" in got:
        e = _errs(got["linewidths"], want["linewidths"], ["linewidths"])
        print(f"{label}: linewidths at {len(Q)} q {e['linewidths']:.2e}")
        assert e["linewidths"] <= 1e-9 and got["linewidths"]["n_imaginary"] == want["linewidths"]["n_imaginary"]
    if "rta" in got:
        e = _errs(got["rta"], want["rta"], ["kappa", "linewidths"])
        print(f"{label}: kappa_RTA {e['kappa']:.2e}, its linewidths {e['linewidths']:.2e}")
        assert e["kappa"] <= 1e-9 and e["linewidths"] <= 1e-9
        assert list(got["rta"]["n_zero_linewidth"]) == list(want["rta"]["n_zero_linewidth"])
    if "lbte" in got:
        e = _errs(got["lbte"], want["lbte"], ["kappa", "kappa_rta"])
        print(f"{label}: kappa_LBTE {e['kappa']:.2e}, kappa_rta {e['kappa_rta']:.2e}; min eigenvalue "
              f"{got['lbte']['min_eigenvalue'].tolist()} 1/ps, dropped {got['lbte']['n_dropped'].tolist()}")
        assert e["kappa"] <= 1e-9 and e["kappa_rta"] <= 1e-9
        assert list(got["lbte"]["n_dropped"]) == list(want["lbte"]["n_dropped"])
    if "spectral" in got:
        e = _errs(got["spectral"], want["spectral"], ["gamma", "delta", "frequency_shifts", "spectral_function"])
        print(f"{label}: spectral_function at {len(SF_Q)} q " + ", ".join(f"{k} {v:.2e}" for k, v in e.items()))
        assert e["gamma"] <= 1e-10 and e["delta"] <= 1e-10 and e["frequency_shifts"] <= 1e-10
        assert e["spectral_function"] <= 3e-9


def test_device_path_matches_spec_path_non_cubic(limno2_fc3, unsplit):
    ph = limno2_fc3
    spec = Phonons(ph.force_constants, ph.cell, fc3=ph.force_constants3, device="cuda", kernels=LbteSpecKernels())
    spec_sf = Phonons(ph.force_constants, ph.cell, fc3=ph.force_constants3, device="cuda",
                      kernels=SpectralFunctionSpecKernels())
    want = _methods(spec, ("linewidths", "rta", "lbte"))
    want.update(_methods(spec_sf, ("spectral",)))
    _check(unsplit, want, f"LiMnO2 2x2x2 on {MESH}, 9 temperatures, device vs specification path")


def _set_chunk(ph, chunk_of, want):
    """Sets ph.ph3_chunk_bytes to the least value at which chunk_of() (q1 per call) is ``want``."""
    lo, hi = 1, Phonons.ph3_chunk_bytes
    while lo < hi:
        ph.ph3_chunk_bytes = (lo + hi) // 2
        lo, hi = (lo, ph.ph3_chunk_bytes) if chunk_of() >= want else (ph.ph3_chunk_bytes + 1, hi)
    ph.ph3_chunk_bytes = lo
    assert chunk_of() == want


def test_split_q1_chunks_match_unsplit(limno2_fc3, unsplit):
    ph = Phonons(limno2_fc3.force_constants, limno2_fc3.cell, fc3=limno2_fc3.force_constants3, device="cuda")
    n_mesh = int(np.prod(MESH))
    chunk = 31  # 72 q1 in calls of 31, 31 and 10
    assert n_mesh // chunk >= 2 and n_mesh % chunk
    _set_chunk(ph, lambda: ph._q1_chunk(len(T9)), chunk)
    got = _methods(ph, ("linewidths", "rta", "lbte"))
    _set_chunk(ph, lambda: ph._spectrum_q1_chunk(len(T9), 201), chunk)
    got.update(_methods(ph, ("spectral",)))
    _check(got, unsplit, f"LiMnO2 2x2x2 on {MESH}, q1 in calls of {chunk} vs unsplit")


def test_temperature_groups_match_unsplit(limno2_fc3, unsplit):
    ph = Phonons(limno2_fc3.force_constants, limno2_fc3.cell, fc3=limno2_fc3.force_constants3, device="cuda")
    m0 = int((unsplit["lbte"]["frequencies"] >= CUT).sum())
    ph.lbte_matrix_bytes = 3 * 8 * m0 * m0  # the 8 temperatures above 0 K in groups of 3, 3 and 2
    got = _methods(ph, ("lbte",))
    _check(got, unsplit, f"LiMnO2 2x2x2 on {MESH}, temperatures in groups of 3 vs one group")


def test_dos_matches_spec_path_non_cubic(limno2_fc3):
    ph = limno2_fc3
    spec = phonon_cells.spec_phonons(ph.force_constants, ph.cell)
    mesh = (9, 7, 5)
    d, ds = ph.dos(mesh, projected=True), spec.dos(mesh, projected=True)
    assert np.abs(d["frequency_points"] - ds["frequency_points"]).max() <= 1e-9 * np.abs(ds["frequency_points"]).max()
    for k in ("total_dos", "integrated_dos", "projected_dos"):
        err = np.abs(d[k] - ds[k]).max() / np.abs(ds[k]).max()
        print(f"LiMnO2 2x2x2 dos {mesh}: {k} vs spec path {err:.2e}")
        assert err <= 1e-9, k
    assert abs(d["integrated_dos"][-1] - 24) <= 1e-12
