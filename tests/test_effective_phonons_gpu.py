"""GPU: the two effective-phonon kernels against their fp64 specification, the replica forces against
predict_structure, and CHGNet.effective_phonons end to end (DESIGN.md section 12.12)."""
import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.phonons import acoustic_sum_rule, effective_force_constants, make_supercell, translation_table
from effective_cells import HarmonicSurrogate
from effective_phonons_kernels import EffectiveSpecKernels
from phonon_cells import model030

pytestmark = pytest.mark.gpu


def _record(name, value):
    """Prints a measured value (run with -s to see it); DESIGN.md section 12.12 quotes them."""
    print(f"MEASURED {name} = {value}")


@pytest.fixture(scope="module")
def cuda_kernels():
    from chgnet_b200._lib import CudaKernels

    return CudaKernels("cuda")


def _random_inputs(m, rng):
    """A LiMnO2 supercell (24 bands), random orthonormal modes, amplitudes, masses, forces and f0."""
    sc = make_supercell(*graphgen.limno2_structure(), m)
    n = len(sc.z)
    e, _ = np.linalg.qr(rng.normal(size=(3 * n, 3 * n)))
    amp = rng.uniform(0.05, 0.3, 3 * n)
    amp[:3] = 0.0
    inv_sqrt_m = 1 / np.sqrt(rng.uniform(5, 60, n))
    lat = np.ascontiguousarray(sc.lattice)
    return sc, [torch.as_tensor(np.ascontiguousarray(x, dtype=np.float64)) for x in
                (e.T, amp, inv_sqrt_m, sc.frac, lat, np.linalg.inv(lat))]


@pytest.mark.parametrize("m", [[4, 4, 4], [[2, 1, 0], [0, 2, 1], [1, 0, 2]]])
def test_kernels_match_specification(cuda_kernels, m):
    rng = np.random.default_rng(0)
    sc, host = _random_inputs(m, rng)
    n, n_s = len(sc.z), 40
    dev = [x.cuda() for x in host]
    frac_d = torch.empty(n_s * n, 3, dtype=torch.float32, device="cuda")
    u_d = torch.empty(n_s, n, 3, dtype=torch.float64, device="cuda")
    cuda_kernels.sample_displacements(*dev, 12345, 2, 7, frac_d, u_d)
    frac_h = torch.empty(n_s * n, 3, dtype=torch.float32)
    u_h = torch.empty(n_s, n, 3, dtype=torch.float64)
    EffectiveSpecKernels().sample_displacements(*host, 12345, 2, 7, frac_h, u_h)
    same = (frac_d.cpu() == frac_h).view(n_s, n, 3).all(-1)  # an fp64 ulp may round a coordinate the other way
    assert (~same).sum() <= max(2, same.numel() // 10000)
    err = float((u_d.cpu() - u_h)[same].abs().max() / u_h.abs().max())
    _record(f"sampler u rel err {m}", err)
    assert err <= 1e-14
    # chunking and repetition: bitwise
    u2 = torch.empty_like(u_d)
    f2 = torch.empty_like(frac_d)
    for s0, s1 in ((0, 13), (13, 14), (14, n_s)):
        cuda_kernels.sample_displacements(*dev, 12345, 2, 7 + s0, f2[s0 * n : s1 * n], u2[s0:s1])
    assert torch.equal(u2, u_d) and torch.equal(f2, frac_d)
    # moments
    perm = torch.as_tensor(translation_table(sc))
    force = torch.as_tensor(rng.normal(size=(n_s, n, 3)))
    f0 = torch.as_tensor(rng.normal(size=(n, 3)))
    n_prim = n // len(sc.points)
    acc_h = torch.zeros(18 * n_prim * n + 2, dtype=torch.float64)
    EffectiveSpecKernels().displacement_moments(u_h, force, f0, perm, acc_h)
    accs = []
    for parts in ([n_s], [1, 16, n_s - 17], [7] * 5 + [n_s - 35]):
        acc = torch.zeros_like(acc_h).cuda()
        s0 = 0
        for p in parts:
            cuda_kernels.displacement_moments(u_h[s0 : s0 + p].cuda(), force[s0 : s0 + p].cuda(), f0.cuda(),
                                              perm.cuda(), acc)
            s0 += p
        accs.append(acc.cpu())
    assert torch.equal(accs[0], accs[1]) and torch.equal(accs[0], accs[2])
    err = float((accs[0] - acc_h).abs().max() / acc_h.abs().max())
    _record(f"moments rel err {m}", err)
    assert err <= 1e-14


@pytest.fixture(scope="module")
def model():
    return model030()


def _limno2_222():
    return make_supercell(*graphgen.limno2_structure(), [2, 2, 2])


def _samples(model, sc, m, t=300.0):
    """m quantum samples at t of the harmonic fc of ``sc`` through the CUDA sampler: (fc, frac [m, N, 3], u)."""
    from chgnet_b200._lib import CudaKernels
    from chgnet_b200.phonons import ATOMIC_MASSES, _expand_compact, sampling_modes

    n = len(sc.z)
    harm = model.phonons(graphgen.limno2_structure(), [2, 2, 2])
    perm = translation_table(sc)
    inv = np.empty_like(perm)
    np.put_along_axis(inv, perm, np.arange(n)[None].repeat(len(perm), 0), axis=1)
    phi = torch.as_tensor(acoustic_sum_rule(harm.force_constants, sc.p2s)[0]).cuda()
    masses = ATOMIC_MASSES[sc.z - 1]
    _, e, amp, _ = sampling_modes(_expand_compact(phi, torch.as_tensor(inv.astype(np.int64)).cuda()), masses, t,
                                  quantum=True, frequency_floor=0.5)
    frac = torch.empty(m * n, 3, dtype=torch.float32, device="cuda")
    u = torch.empty(m, n, 3, dtype=torch.float64, device="cuda")
    lat = np.ascontiguousarray(sc.lattice)
    CudaKernels("cuda").sample_displacements(e, amp, torch.as_tensor(1 / np.sqrt(masses)).cuda(),
                                             torch.as_tensor(sc.frac).cuda(), torch.as_tensor(lat).cuda(),
                                             torch.as_tensor(np.linalg.inv(lat)).cuda(), 0, 0, 0, frac, u)
    return harm.force_constants, frac.view(m, n, 3).double(), u


def test_replica_forces_match_predict_structure(model):
    """Forces and energies of 300 K samples through the replica batches against predict_structure, whose graph is
    built on the device, one structure at a time."""
    from chgnet_b200.model import _ReplicaForces

    sc = _limno2_222()
    n, m = len(sc.z), 8
    _, frac, u = _samples(model, sc, m)
    f, en = _ReplicaForces(model, sc)(frac)
    x = frac.cpu().numpy()
    f_err = e_err = 0.0
    for s in range(m):
        ref = model.predict_structure((sc.z, x[s], sc.lattice), task="ef")
        f_err = max(f_err, float(np.abs(f[s].cpu().numpy() - ref["f"]).max()))
        e_err = max(e_err, abs(float(en[s]) / n - float(ref["e"])))
    _record("300 K max |u| (A)", float(u.norm(dim=-1).max()))
    _record("replica vs predict_structure max |dF| (eV/A)", f_err)
    _record("replica vs predict_structure max |dE| (eV/atom)", e_err)
    assert f_err <= 2e-4 and e_err <= 2e-6


def test_harmonic_surrogate_through_device_path():
    """Random bond springs on LiMnO2 2x2x2 (unequal masses): symmetric, translation-invariant force constants that
    obey the acoustic sum rule, as real ones do.  One iteration through the CUDA kernels recovers them."""
    sc = _limno2_222()
    rng = np.random.default_rng(3)
    n = len(sc.z)
    perm = translation_table(sc)
    full = np.zeros((n, n, 3, 3))
    for k in range(len(sc.p2s)):
        for j in rng.choice(n, 6, replace=False):
            a = rng.normal(size=(3, 3))
            kk = a @ a.T + np.eye(3)
            for l in range(len(perm)):
                i, jl = perm[l, sc.p2s[k]], perm[l, j]
                if i == jl:
                    continue
                full[i, jl] -= kk
                full[jl, i] -= kk
                full[i, i] += kk
                full[jl, jl] += kk
    fc = np.ascontiguousarray(full[sc.p2s])
    sur = HarmonicSurrogate(sc, fc, rng.normal(size=(n, 3)) * 0.05)

    def forces(frac):
        f, e = sur(frac.cpu())
        return f.cuda(), e.cuda()

    out, info = effective_force_constants(forces, sc, fc, 300.0, device="cuda", n_samples=64, n_iterations=1,
                                          batch_size=3)
    ref = acoustic_sum_rule(fc, sc.p2s)[0]
    err = float(np.abs(out - ref).max() / np.abs(ref).max())
    _record("device harmonic surrogate rel err", err)
    assert err <= 1e-10


def test_low_temperature_limit(model):
    """Classical 1 K: the effective fc equals the harmonic fc within the statistical bound."""
    s = graphgen.limno2_structure()
    ph = model.effective_phonons(s, [2, 2, 2], 1.0, quantum=False, n_samples=64, n_iterations=1, seed=1)
    harm = ph.effective["harmonic_force_constants"]
    ref = acoustic_sum_rule(harm, _limno2_222().p2s)[0]
    dev = float(np.abs(ph.force_constants - ref).max())
    _record("1 K classical max |Phi_eff - Phi_harm| (eV/A^2)", dev)
    _record("1 K sigma_a", ph.effective["sigma_a"])
    # fp32 forces of displacements of ~0.005 A: the harmonic fit is limited by the forces' rounding and the
    # anharmonicity at that amplitude, both far below the fc scale (~10 eV/A^2)
    assert dev <= 0.05 * float(np.abs(ref).max())


def test_room_temperature_run(model):
    """A 300 K quantum run is finite, its history has the stated keys, and two runs agree.  The samples and moments
    are bitwise reproducible (test_kernels_match_specification), but the engine's forces and Hessian-vector products
    are not: they differ between calls by ~1e-14 eV/A, which three iterations amplify."""
    s = graphgen.limno2_structure()
    a = model.effective_phonons(s, [2, 2, 2], 300.0, n_samples=128, n_iterations=3, seed=0)
    b = model.effective_phonons(s, [2, 2, 2], 300.0, n_samples=128, n_iterations=3, seed=0)
    assert np.all(np.isfinite(a.force_constants))
    assert [set(h) for h in a.effective["history"]] == [{"max_change", "n_imaginary", "sigma_a", "u0"}] * 3
    diff = float(np.abs(a.force_constants - b.force_constants).max())
    _record("effective_phonons twice bitwise equal", bool(np.array_equal(a.force_constants, b.force_constants)))
    _record("effective_phonons twice max |dPhi| (eV/A^2)", diff)
    assert diff <= 1e-4
    harm = a.__class__(a.effective["harmonic_force_constants"], a.cell)
    n_h = harm.thermal_properties([8, 8, 8], [300.0])["n_imaginary"]
    n_e = a.thermal_properties([8, 8, 8], [300.0])["n_imaginary"]
    _record("300 K history", a.effective["history"])
    _record("n_imaginary on 8^3 mesh harmonic -> effective", [n_h, n_e])
