"""-m gpu: device-resident MD / relaxation (chgnet_b200/dynamics_device.py, SURVEY.md §8 row f2) against the host
drivers of chgnet_b200/dynamics.py (the restatement of what ase + CHGNetCalculator do in the reference,
chgnet/model/dynamics.py:129-181) and against itself without the Verlet skin."""
import os

import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from chgnet_b200.model import CHGNet

    path = os.path.join(os.path.dirname(__file__), "golden", "chgnet_0.3.0_weights.npz")
    return CHGNet.from_file(path, version="0.3.0").to("cuda")


def _system(seed=4200, rattle=0.03):
    z, frac, lat = graphgen.limno2_structure((2, 2, 1), rattle, seed)
    return z, frac @ lat, lat


def test_device_trajectory_equals_the_host_driver_and_conserves_energy(model):
    from chgnet_b200.dynamics import Atoms, CHGNetCalculator, VelocityVerlet
    from chgnet_b200.dynamics_device import DeviceMD

    z, pos, cell = _system()
    steps = 50
    host_atoms = Atoms(z, pos, cell)
    host = VelocityVerlet(host_atoms, CHGNetCalculator(model=model, on_isolated_atoms="ignore"), timestep=2.0)
    host.set_temperature(300.0, seed=7)
    v0 = host_atoms.velocities.copy()
    dev = DeviceMD(model, z, pos, cell, timestep=2.0, velocities=v0, skin=0.5)
    wide = DeviceMD(model, z, pos, cell, timestep=2.0, velocities=v0, skin=1.2, use_cuda_graph=False)  # different lists, same physics
    exact = DeviceMD(model, z, pos, cell, timestep=2.0, velocities=v0, skin=0.0)  # exact lists rebuilt on the device every step
    e0 = host.potential_energy() + host.kinetic_energy()
    hlog = host.run(steps)
    dlog = dev.run(steps)
    wide.run(steps)
    exact.run(steps)
    de = np.abs(exact.positions() - host_atoms.positions).max()
    assert de < 1e-4 and exact.n_builds == steps + 1, (de, exact.n_builds)
    dx = np.abs(dev.positions() - host_atoms.positions).max()
    dn = np.abs(dev.positions() - wide.positions()).max()
    print(f"50 steps: max |x_device - x_host (graph rebuilt every step)| = {dx:.2e} A, |x_skin0.5 - x_skin1.2| = {dn:.2e} A; "
          f"graph builds: skin 0.5 {dev.n_builds}, skin 1.2 {wide.n_builds}, host {steps + 1}")
    assert dx < 1e-4 and dn < 1e-4
    assert wide.n_builds <= dev.n_builds < 12  # the skin really avoids rebuilds
    for h, d in zip(hlog[::10], dlog[::10]):
        assert abs(h["e_pot"] - d["e_pot"]) < 1e-3 and abs(h["e_kin"] - d["e_kin"]) < 1e-3
    drift = max(abs(d["e_pot"] + d["e_kin"] - e0) for d in dlog)
    print(f"NVE total-energy drift over {steps} steps of 2 fs: {drift:.2e} eV ({len(z)} atoms)")
    assert drift < 2e-2
    assert dlog[-1]["temperature"] > 10.0


def test_cuda_graph_step_equals_the_eager_step(model):
    from chgnet_b200.dynamics_device import DeviceMD

    z, pos, cell = _system(4201)
    a = DeviceMD(model, z, pos, cell, timestep=1.0, skin=0.6, use_cuda_graph=True)
    b = DeviceMD(model, z, pos, cell, timestep=1.0, skin=0.6, use_cuda_graph=False)
    for md in (a, b):
        md.set_temperature(500.0, seed=3)
    a.run(12, log_every=0)
    b.run(12, log_every=0)
    assert np.abs(a.positions() - b.positions()).max() < 1e-9
    assert abs(a.potential_energy - b.potential_energy) < 1e-7


def test_device_fire_relaxes(model):
    from chgnet_b200.dynamics_device import DeviceFIRE

    z, pos, cell = _system(4202)
    fire = DeviceFIRE(model, z, pos, cell)
    e_start = fire.potential_energy
    f_start = float(fire.f.pow(2).sum(dim=1).max().sqrt())
    res = fire.run(fmax=0.05, steps=300)
    print(f"FIRE: {res['steps']} steps, fmax {f_start:.3f} -> {res['fmax']:.3f} eV/A, E {e_start:.4f} -> {fire.potential_energy:.4f} eV, "
          f"{res['graph_builds']} graph builds")
    assert res["fmax"] < f_start and fire.potential_energy < e_start
    assert res["converged"]


def test_device_fire_follows_fire_relax(model, monkeypatch):
    """DeviceFIRE and the host fire_relax take the same 30 FIRE steps from a hard rattle; the 0.2 A step limit is
    active on some of them (seen through fire_update on the host trajectory)."""
    from chgnet_b200 import dynamics
    from chgnet_b200.dynamics import Atoms, CHGNetCalculator, fire_relax
    from chgnet_b200.dynamics_device import DeviceFIRE

    steps, dt0 = 30, 0.4
    z, pos, cell = _system(4203, rattle=0.1)
    spec, clamped = dynamics.fire_update, []

    def recording_update(x, v, f, state, dt_max, max_step):
        out = spec(x, v, f, state, dt_max, max_step)
        clamped.append(bool(np.sqrt(((out[2][0] * out[1]) ** 2).sum(axis=1)).max() > max_step))
        return out

    monkeypatch.setattr(dynamics, "fire_update", recording_update)
    host_atoms = Atoms(z, pos, cell)
    fire_relax(host_atoms, CHGNetCalculator(model=model, on_isolated_atoms="ignore"), fmax=0.0, steps=steps, dt=dt0)
    dev = DeviceFIRE(model, z, pos, cell, dt=dt0)
    res = dev.run(fmax=0.0, steps=steps)
    dx = np.abs(dev.positions() - host_atoms.positions).max()
    print(f"FIRE {steps} steps: max |x_DeviceFIRE - x_fire_relax| = {dx:.2e} A; step limit active on steps "
          f"{[i for i, c in enumerate(clamped) if c]}")
    assert len(clamped) == steps and res["steps"] == steps and any(clamped)
    assert dx < 1e-4
