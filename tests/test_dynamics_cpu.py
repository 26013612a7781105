"""CPU: the calculator shim and the host MD / relaxation drivers (reference chgnet/model/dynamics.py:58-181)
with the torch kernel specifications injected in place of the CUDA library."""
import os

import numpy as np
import pytest

from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch  # noqa: F401
from chgnet_b200.dynamics import GPA, Atoms, CHGNetCalculator, VelocityVerlet, fire_relax, fire_update
from chgnet_b200.engine import Engine
from chgnet_b200.weights import pack_weights
from oracle.kernel_specs import SpecKernels


@pytest.fixture()
def calc(monkeypatch):
    from chgnet_b200.model import CHGNet

    path = os.path.join(os.path.dirname(__file__), "golden", "chgnet_0.3.0_weights.npz")
    model = CHGNet.from_file(path, version="0.3.0")
    eng = Engine(pack_weights(model.state_dict(), model.model_args, device="cpu"), SpecKernels())
    monkeypatch.setattr(model, "_get_engine", lambda: eng)
    monkeypatch.setenv("CHGNET_B200_ENGINE", "python")
    return CHGNetCalculator(model=model, return_site_energies=True)


def _limno2(displacement=0.0, seed=0):
    z, frac, lat = graphgen.limno2_structure((1, 1, 1), displacement, seed)
    return Atoms(z, frac @ lat, lat)


def test_calculator_results_follow_the_reference_conventions(calc, golden):
    atoms = _limno2()
    calc.calculate(atoms)
    r = calc.results
    assert r["energy"] == pytest.approx(-7.36769 * 8, abs=1e-3) and r["free_energy"] == r["energy"]  # tests/test_model.py:68, extensive
    assert r["forces"].shape == (8, 3) and r["stress"].shape == (3, 3) and r["magmoms"].shape == (8,)
    assert np.allclose(r["stress"], golden["limno2.ref32.s"] * GPA, atol=2e-3 * GPA)  # GPa -> eV/A^3 (dynamics.py:69)
    assert np.allclose(r["forces"], golden["limno2.ref32.f"], atol=1e-3)
    assert r["energies"].shape == (8,) and r["crystal_fea"].shape == (64,)
    assert calc.n_params == 412525 and calc.version == "0.3.0"
    calc.calculate(atoms, task="e")
    assert "energy" in calc.results


def test_relaxation_and_nve_dynamics(calc):
    atoms = _limno2(0.04, seed=3)
    calc.calculate(atoms, task="ef")
    e0, f0 = float(calc.results["energy"]), float(np.abs(calc.results["forces"]).max())
    out = fire_relax(atoms, calc, fmax=0.02, steps=12)
    assert out["energies"][-1] < e0 - 1e-4 and out["fmax"] < f0  # downhill
    md_atoms = _limno2(0.02, seed=5)
    md = VelocityVerlet(md_atoms, calc, timestep=1.0)
    md.set_temperature(300.0, seed=1)
    e_start = md.potential_energy() + md.kinetic_energy()
    log = md.run(6)
    e_end = log[-1]["e_pot"] + log[-1]["e_kin"]
    assert abs(e_end - e_start) < 5e-3, (e_start, e_end)  # eV for 8 atoms over 6 fs
    assert 50 < log[-1]["temperature"] < 1000 and md.nsteps == 6


def _fire_relax_as_written_before_fire_update(atoms, calculator, fmax, steps, dt, dt_max):
    """fire_relax as it was before its update was factored out into fire_update (the regression reference)."""
    n_min, f_inc, f_dec, alpha_start, f_alpha = 5, 1.1, 0.5, 0.1, 0.99
    v = np.zeros_like(atoms.positions)
    alpha, n_pos = alpha_start, 0
    energies = []
    for step in range(steps):
        calculator.calculate(atoms, task="ef")
        f = np.asarray(calculator.results["forces"], dtype=np.float64)
        energies.append(float(calculator.results["energy"]))
        fnorm = float(np.sqrt((f**2).sum(axis=1)).max())
        if fnorm < fmax:
            break
        power = float((f * v).sum())
        if power > 0:
            v = (1 - alpha) * v + alpha * f * np.linalg.norm(v) / max(np.linalg.norm(f), 1e-30)
            n_pos += 1
            if n_pos > n_min:
                dt, alpha = min(dt * f_inc, dt_max), alpha * f_alpha
        else:
            v[:] = 0.0
            dt, alpha, n_pos = dt * f_dec, alpha_start, 0
        v = v + dt * f
        dr = dt * v
        norm = np.sqrt((dr**2).sum(axis=1)).max()
        if norm > 0.2:
            dr *= 0.2 / norm
        atoms.positions = atoms.positions + dr
    return {"energies": energies, "fmax": fnorm, "steps": step + 1, "converged": fnorm < fmax}


class _ScriptedForces:
    """A calculator that returns the next force array of a fixed script, whatever the positions."""

    def __init__(self, forces) -> None:
        self.forces, self.k, self.results = forces, 0, {}

    def calculate(self, atoms, task="ef") -> None:
        self.results = {"forces": self.forces[self.k], "energy": float(self.k)}
        self.k += 1


def test_fire_update_reproduces_the_previous_fire_relax_bitwise():
    rng = np.random.default_rng(11)
    direction = rng.normal(size=(8, 3))
    # mostly along one direction with a slowly turning amplitude: downhill runs, sign changes of f.v (resets) and
    # steps beyond 0.2 A
    script = [(20.0 * np.cos(0.3 * k) + 2.5) * direction + 1.5 * rng.normal(size=(8, 3)) for k in range(60)]
    runs, starts = [], []
    for relax in (_fire_relax_as_written_before_fire_update, fire_relax):
        atoms = _limno2(0.04, seed=3)
        x_start = atoms.positions.copy()
        out = relax(atoms, _ScriptedForces(script), fmax=1e-3, steps=60, dt=0.1, dt_max=0.6)
        runs.append((atoms.positions, out))
        starts.append(x_start)
    (x_old, out_old), (x_new, out_new) = runs
    assert np.array_equal(x_old, x_new) and out_old == out_new
    # the script reaches the step limit: replay it through fire_update and look at the unscaled steps
    x, v, state, clamped, resets = starts[1], np.zeros((8, 3)), (0.1, 0.1, 0), 0, 0
    for f in script:
        x_next, v, new_state = fire_update(x, v, f, state, 0.6)
        clamped += int(np.sqrt(((new_state[0] * v) ** 2).sum(axis=1)).max() > 0.2)
        resets += int(new_state[2] == 0 and state[2] > 0)
        x, state = x_next, new_state
    assert np.array_equal(x, x_new) and clamped > 0 and resets > 0, (clamped, resets)


def test_fire_schedule_follows_the_sign_of_the_power():
    """dt, alpha and the downhill count for a scripted sign of f.v (n_min = 5, f_inc 1.1, f_dec 0.5, f_alpha 0.99)."""
    f = np.ones((2, 3))
    signs = [0, +1, +1, +1, +1, +1, +1, +1, +1, -1, +1, 0]
    table = [  # (dt, alpha, n_pos) after each step; dt_max = 0.06
        (0.1 * 0.5, 0.1, 0),  # v = 0: uphill
        (0.05, 0.1, 1), (0.05, 0.1, 2), (0.05, 0.1, 3), (0.05, 0.1, 4), (0.05, 0.1, 5),
        (0.05 * 1.1, 0.1 * 0.99, 6),  # more than n_min downhill steps in a row: grow dt, decay alpha
        (0.06, 0.1 * 0.99 * 0.99, 7),  # 0.0605 is capped at dt_max
        (0.06, 0.1 * 0.99 * 0.99 * 0.99, 8),
        (0.06 * 0.5, 0.1, 0),  # uphill: halve dt, reset alpha and the count
        (0.03, 0.1, 1),
        (0.03 * 0.5, 0.1, 0),  # f.v = 0 counts as uphill
    ]
    state = (0.1, 0.1, 0)
    for sign, want in zip(signs, table):
        _, _, state = fire_update(np.zeros((2, 3)), sign * f, f, state, dt_max=0.06)
        assert state == want, (sign, state, want)
        assert type(state[2]) is int


def test_fire_step_limit_scales_the_whole_update():
    """Steps of 0.4 A and 0.1 A become 0.2 A and 0.05 A: one scale for all atoms, directions kept, v not scaled."""
    f = np.array([[0.4, 0.0, 0.0], [0.0, 0.1, 0.0]])
    x, v, state = fire_update(np.zeros((2, 3)), np.zeros((2, 3)), f, (2.0, 0.1, 0))  # uphill: dt = 1, dr = f
    assert state == (1.0, 0.1, 0)
    assert np.array_equal(x, [[0.2, 0.0, 0.0], [0.0, 0.05, 0.0]])
    assert np.array_equal(v, f)
    x, _, _ = fire_update(np.zeros((2, 3)), np.zeros((2, 3)), f, (2.0, 0.1, 0), max_step=0.5)  # below the limit
    assert np.array_equal(x, f)


def test_isolated_atoms_policy(calc):
    atoms = Atoms([3, 8], [[0.0, 0, 0], [10.0, 10, 10]], np.eye(3) * 20.0)  # both atoms isolated: no edges at all
    calc.calculate(atoms, task="e")  # nothing to warn about when the graph has no edges (model.py:841-843)
    far = Atoms([3, 8, 8], [[0.0, 0, 0], [1.5, 0, 0], [10.0, 10, 10]], np.eye(3) * 20.0)
    with pytest.warns(UserWarning, match="isolated atoms"):
        calc.calculate(far, task="e")
    calc.on_isolated_atoms = "error"
    with pytest.raises(ValueError):
        calc.calculate(far, task="e")
