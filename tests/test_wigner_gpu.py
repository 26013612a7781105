"""-m gpu: the Wigner coherence conductivity on the device (Phonons.thermal_conductivity_wigner).

* ``chg_coherence_conductivity`` against its fp64 specification (tests/wigner_kernels.py, run with torch on the same
  device) on random unitary eigenvectors, random Hermitian dD/dQ, frequencies with negative, sub-cutoff and exactly
  degenerate values and linewidths with zeros and negatives, at 5 temperatures (a ragged temperature tile): 24 bands on
  512 q and 93 bands on 64 q; two calls bitwise equal, q-chunked calls against one call;
* on the device fc3 of LiMnO2 2x2x2, ``thermal_conductivity_wigner`` on 6^3 at 0, 300 and 1 000 K against the
  specification path, and its kappa_p bitwise ``thermal_conductivity``'s kappa."""
import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.phonons import THERMAL_CUTOFF_THZ, Phonons, _degenerate_set_ids
from wigner_kernels import WignerSpecKernels

pytestmark = pytest.mark.gpu
CUT = THERMAL_CUTOFF_THZ


def _random_inputs(n_q, nb, n_t, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    f64, dev = torch.float64, "cuda"
    nu = torch.rand(n_q, nb, generator=g, device=dev, dtype=f64) * 23.0 - 3.0
    nu[:, 0] = 0.0
    nu[::3, 1] = 5e-4
    nu[1::3, 1] = CUT
    nu[2::3, 1] = -1e-2
    nu = torch.sort(nu, dim=1)[0]
    nu[:, nb // 2 + 1] = nu[:, nb // 2]  # exactly degenerate pairs
    nu[:, nb - 1] = nu[:, nb - 2] = nu[:, nb - 3]
    nu = nu.contiguous()
    a = torch.randn(n_q, nb, nb, generator=g, device=dev, dtype=f64) + 1j * torch.randn(
        n_q, nb, nb, generator=g, device=dev, dtype=f64)
    e = torch.linalg.qr(a)[0].mT.contiguous()
    d = torch.randn(n_q, 3, nb, nb, generator=g, device=dev, dtype=f64) + 1j * torch.randn(
        n_q, 3, nb, nb, generator=g, device=dev, dtype=f64)
    d = (0.5 * (d + d.mH)).contiguous()
    sid = _degenerate_set_ids(nu).to(torch.int32)
    cv = torch.rand(n_t, n_q, nb, generator=g, device=dev, dtype=f64) * 8.6e-5
    cv[0] = 0.0  # T = 0
    gamma = torch.rand(n_t, n_q, nb, generator=g, device=dev, dtype=f64) * 0.5
    gamma[..., ::7] = 0.0
    gamma[..., 3::11] = -0.1
    return nu, e, d, sid, cv.contiguous(), gamma.contiguous()


@pytest.mark.parametrize("n_q,nb", [(512, 24), (64, 93)])
def test_kernel_matches_spec(n_q, nb):
    from chgnet_b200._lib import CudaKernels

    n_t = 5
    nu, e, d, sid, cv, gamma = _random_inputs(n_q, nb, n_t, seed=nb + n_q)
    kern, spec = CudaKernels("cuda"), WignerSpecKernels()

    def run(k, step=n_q):
        out = torch.zeros(n_t, 3, 3, dtype=torch.float64, device="cuda")
        for s in range(0, n_q, step):
            sl = slice(s, s + step)
            k.coherence_conductivity(nu[sl], e[sl], d[sl], sid[sl], cv[:, sl].contiguous(), gamma[:, sl].contiguous(),
                                     CUT, out)
        return out

    got, again, want = run(kern), run(kern), run(spec)
    assert torch.equal(got, again)
    chunked = run(kern, 37)
    scale = float(want.abs().max())
    err = float((got - want).abs().max()) / scale
    err_chunk = float((chunked - got).abs().max()) / scale
    print(f"{nb} bands on {n_q} q, 5 temperatures: kernel vs specification {err:.2e} of max|kappa| {scale:.3e}; "
          f"bitwise reproducible; 37-q calls vs one call {err_chunk:.2e}")
    assert scale > 0 and torch.all(got[0] == 0)
    assert err <= 5e-15 and err_chunk <= 5e-15  # measured 6.4e-16 and 3.7e-16 on an H100


@pytest.fixture(scope="module")
def limno2_fc3():
    model = phonon_cells.model030()
    return model.phonons(graphgen.limno2_structure(), [2, 2, 2], third_order=True)


def test_device_path_matches_spec_path(limno2_fc3):
    ph = limno2_fc3
    spec = Phonons(ph.force_constants, ph.cell, fc3=ph.force_constants3, device="cuda", kernels=WignerSpecKernels())
    mesh, temps = (6, 6, 6), [0.0, 300.0, 1000.0]
    got, want = ph.thermal_conductivity_wigner(mesh, temps), spec.thermal_conductivity_wigner(mesh, temps)
    rta = ph.thermal_conductivity(mesh, temps)
    err_c = np.abs(got["kappa_c"] - want["kappa_c"]).max() / np.abs(want["kappa_c"]).max()
    err_p = np.abs(got["kappa_p"] - want["kappa_p"]).max() / np.abs(want["kappa_p"]).max()
    print(f"LiMnO2 2x2x2 Wigner on 6^3 at 0, 300, 1000 K: device vs specification path kappa_C {err_c:.2e}, kappa_P "
          f"{err_p:.2e}; 300 K diagonal kappa_P {np.diag(got['kappa_p'][1])}, kappa_C {np.diag(got['kappa_c'][1])} "
          f"W/(m K); 1000 K kappa_P {np.diag(got['kappa_p'][2])}, kappa_C {np.diag(got['kappa_c'][2])}")
    assert np.array_equal(got["kappa_p"], rta["kappa"])
    assert np.array_equal(got["kappa"], got["kappa_p"] + got["kappa_c"])
    assert np.all(got["kappa_c"][0] == 0)
    # measured 2.2e-14 and 1.3e-14 on an H100: the linewidths of the two paths agree to ~1e-14 here
    assert err_c <= 1e-12 and err_p <= 1e-12
