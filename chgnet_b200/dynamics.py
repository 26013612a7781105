"""Calculator shim and minimal host-side MD / relaxation drivers (SURVEY.md §8 row f2, host stage).

``CHGNetCalculator`` mirrors the reference's ASE calculator (chgnet/model/dynamics.py:58-181): same
constructor keywords, ``calculate(atoms, properties, system_changes, task)``, the same ``results`` keys
and unit conventions (total energy in eV, forces in eV/A, stress x ``stress_weight`` = eV/A^3 as a 3x3
array, ``magmoms``, ``free_energy``, ``crystal_fea``, optional ``energies``).  When ``ase`` is installed
it subclasses ``ase.calculators.calculator.Calculator`` and can be attached to ``ase.Atoms``; without
``ase`` it is a plain object that accepts anything with ``get_atomic_numbers() / get_positions() /
get_cell()`` (e.g. :class:`Atoms` below), so ``VelocityVerlet`` and ``fire_relax`` here run stand-alone.

Every step rebuilds the graph with the native host builder (``chg_graph_build``) and runs one
``chg_forward``; keeping positions / velocities on the device and building the graph there is the next
stage of this row.
"""
from __future__ import annotations

import numpy as np

from chgnet_b200 import PredTask

GPA = 1.0 / 160.21766208  # GPa -> eV/A^3 (ase.units.GPa)
FS = 0.09822694788464063  # fs in ASE time units (A sqrt(amu/eV))  (ase.units.fs)
KB = 8.617333262e-5  # eV/K

# standard atomic weights, Z = 1..94 (amu)
ATOMIC_MASSES = np.array([
    1.008, 4.002602, 6.94, 9.0121831, 10.81, 12.011, 14.007, 15.999, 18.998403163, 20.1797, 22.98976928, 24.305, 26.9815385,
    28.085, 30.973761998, 32.06, 35.45, 39.948, 39.0983, 40.078, 44.955908, 47.867, 50.9415, 51.9961, 54.938044, 55.845,
    58.933194, 58.6934, 63.546, 65.38, 69.723, 72.630, 74.921595, 78.971, 79.904, 83.798, 85.4678, 87.62, 88.90584, 91.224,
    92.90637, 95.95, 97.90721, 101.07, 102.90550, 106.42, 107.8682, 112.414, 114.818, 118.710, 121.760, 127.60, 126.90447,
    131.293, 132.90545196, 137.327, 138.90547, 140.116, 140.90766, 144.242, 144.91276, 150.36, 151.964, 157.25, 158.92535,
    162.500, 164.93033, 167.259, 168.93422, 173.054, 174.9668, 178.49, 180.94788, 183.84, 186.207, 190.23, 192.217, 195.084,
    196.966569, 200.592, 204.38, 207.2, 208.98040, 208.98243, 209.98715, 222.01758, 223.01974, 226.02541, 227.02775, 232.0377,
    231.03588, 238.02891, 237.04817, 244.06421])

try:  # optional: real ASE base class
    from ase.calculators.calculator import Calculator as _Base
    from ase.calculators.calculator import all_changes, all_properties
except ImportError:  # stand-alone
    all_changes, all_properties = ["positions", "numbers", "cell", "pbc"], ["energy", "forces", "stress", "magmoms"]

    class _Base:  # the two things the shim needs from ase's Calculator
        def __init__(self, **_: object) -> None:
            self.results: dict = {}
            self.atoms = None

        def calculate(self, atoms=None, properties=None, system_changes=None) -> None:
            if atoms is not None:
                self.atoms = atoms


class Atoms:
    """Minimal periodic structure (numbers, Cartesian positions in A, cell rows = lattice vectors)."""

    def __init__(self, numbers, positions, cell, velocities=None) -> None:
        self.numbers = np.asarray(numbers, dtype=np.int64)
        self.positions = np.asarray(positions, dtype=np.float64).reshape(-1, 3)
        self.cell = np.asarray(cell, dtype=np.float64).reshape(3, 3)
        self.velocities = np.zeros_like(self.positions) if velocities is None else np.asarray(velocities, dtype=np.float64)
        self.calc = None

    def get_atomic_numbers(self):
        return self.numbers

    def get_positions(self):
        return self.positions

    def get_cell(self):
        return self.cell

    def get_masses(self):
        return ATOMIC_MASSES[self.numbers - 1]

    def __len__(self) -> int:
        return len(self.numbers)


class CHGNetCalculator(_Base):
    """CHGNet calculator (reference dynamics.py:58-181) on the H100 kernel path."""

    implemented_properties = ("energy", "forces", "stress", "magmoms", "energies")

    def __init__(self, model=None, *, use_device: str | None = None, check_cuda_mem: bool = False,
                 stress_weight: float = GPA, on_isolated_atoms: str = "warn", return_site_energies: bool = False,
                 **kwargs) -> None:
        super().__init__(**kwargs)
        from chgnet_b200.model import CHGNet

        self.model = model if model is not None else CHGNet.load(use_device=use_device, verbose=False)
        if use_device is not None:
            self.model = self.model.to(use_device)
        self.device = self.model.device
        self.stress_weight = stress_weight
        self.return_site_energies = return_site_energies
        self.on_isolated_atoms = on_isolated_atoms
        del check_cuda_mem

    @classmethod
    def from_file(cls, path: str, use_device: str | None = None, **kwargs):
        from chgnet_b200.model import CHGNet

        return cls(model=CHGNet.from_file(path), use_device=use_device, **kwargs)

    @property
    def version(self) -> str | None:
        return self.model.version

    @property
    def n_params(self) -> int:
        return self.model.n_params

    def calculate(self, atoms=None, properties=None, system_changes=None, task: PredTask = "efsm") -> None:
        properties = properties or all_properties
        system_changes = system_changes or all_changes
        super().calculate(atoms=atoms, properties=properties, system_changes=system_changes)
        atoms = atoms if atoms is not None else self.atoms
        numbers = np.asarray(atoms.get_atomic_numbers())
        cell = np.asarray(atoms.get_cell(), dtype=np.float64).reshape(3, 3)
        frac = np.asarray(atoms.get_positions(), dtype=np.float64) @ np.linalg.inv(cell)
        from chgnet_b200 import graphgen

        graph = graphgen.make_crystal_graph(numbers, frac, cell, atom_graph_cutoff=self.model.graph_converter.atom_graph_cutoff,
                                            bond_graph_cutoff=self.model.graph_converter.bond_graph_cutoff)
        if self.on_isolated_atoms != "ignore":
            centers = graph.atom_graph[:, 0].tolist() if graph.atom_graph.dim() == 2 else []
            isolated = set(range(len(numbers))) - set(centers)
            if isolated:
                msg = f"structure has isolated atoms {sorted(isolated)} (no neighbour within the atom-graph cutoff)"
                if self.on_isolated_atoms == "error":
                    raise ValueError(msg)
                import warnings

                warnings.warn(msg, stacklevel=2)
        pred = self.model.predict_graph(graph, task=task, return_crystal_feas=True,
                                        return_site_energies=self.return_site_energies)
        extensive = len(numbers) if self.model.is_intensive else 1
        key_map = {"e": ("energy", extensive), "f": ("forces", 1), "m": ("magmoms", 1), "s": ("stress", self.stress_weight)}
        self.results = {**getattr(self, "results", {}),
                        **{long: pred[k] * fac for k, (long, fac) in key_map.items() if k in pred}}
        self.results["free_energy"] = self.results["energy"]
        self.results["crystal_fea"] = pred["crystal_fea"]
        if self.return_site_energies:
            self.results["energies"] = pred["site_energies"]

    def get_hessian(self, atoms=None):
        """``[3N,3N]`` Hessian d^2E/dx dx of the total energy at fixed cell, in eV/A^2 (``CHGNet.predict_hessian``)."""
        atoms = atoms if atoms is not None else self.atoms
        cell = np.asarray(atoms.get_cell(), dtype=np.float64).reshape(3, 3)
        frac = np.asarray(atoms.get_positions(), dtype=np.float64) @ np.linalg.inv(cell)
        return self.model.predict_hessian((np.asarray(atoms.get_atomic_numbers()), frac, cell))


class VelocityVerlet:
    """NVE molecular dynamics on the host (the integrator of ase.md.verlet restated): one calculator
    call per step.  ``timestep`` in fs."""

    def __init__(self, atoms, calculator: CHGNetCalculator, timestep: float = 2.0, task: PredTask = "ef") -> None:
        self.atoms, self.calc, self.dt, self.task = atoms, calculator, timestep * FS, task
        self.calc.calculate(atoms, task=task)
        self.forces = np.asarray(self.calc.results["forces"], dtype=np.float64)
        self.nsteps = 0

    def kinetic_energy(self) -> float:
        return float(0.5 * (self.atoms.get_masses()[:, None] * self.atoms.velocities**2).sum())

    def potential_energy(self) -> float:
        return float(self.calc.results["energy"])

    def temperature(self) -> float:
        return 2.0 * self.kinetic_energy() / (3.0 * len(self.atoms) * KB)

    def set_temperature(self, kelvin: float, seed: int = 0) -> None:
        rng = np.random.default_rng(seed)
        m = self.atoms.get_masses()[:, None]
        v = rng.normal(size=self.atoms.positions.shape) * np.sqrt(KB * kelvin / m)
        v -= (m * v).sum(axis=0) / m.sum()  # no centre-of-mass drift
        self.atoms.velocities = v

    def run(self, steps: int) -> list[dict]:
        log = []
        m = self.atoms.get_masses()[:, None]
        for _ in range(steps):
            self.atoms.velocities = self.atoms.velocities + 0.5 * self.dt * self.forces / m
            self.atoms.positions = self.atoms.positions + self.dt * self.atoms.velocities
            self.calc.calculate(self.atoms, task=self.task)
            self.forces = np.asarray(self.calc.results["forces"], dtype=np.float64)
            self.atoms.velocities = self.atoms.velocities + 0.5 * self.dt * self.forces / m
            self.nsteps += 1
            log.append({"step": self.nsteps, "e_pot": self.potential_energy(), "e_kin": self.kinetic_energy(),
                        "temperature": self.temperature()})
        return log


FIRE_N_MIN, FIRE_F_INC, FIRE_F_DEC, FIRE_ALPHA_START, FIRE_F_ALPHA = 5, 1.1, 0.5, 0.1, 0.99


def fire_update(x, v, f, state, dt_max: float = 1.0, max_step: float = 0.2):
    """One FIRE update (Bitzek et al. 2006) in fp64: the specification of ``fire_relax`` and of ``chg_fire_step``.

    ``x, v, f`` are [N, 3] positions, velocities and forces; ``state = (dt, alpha, n_pos)``.  A step with
    power f.v > 0 mixes v towards f, counts itself downhill and, after more than ``n_min`` downhill steps in a row,
    grows dt (capped at ``dt_max``) and decays alpha; any other step (v = 0 included) zeroes v, halves dt and resets
    alpha and the count.  Then v += dt f and dr = dt v; when the largest per-atom step max_i |dr_i| exceeds
    ``max_step`` the whole dr is scaled by ``max_step / max_i |dr_i|``, so every atom keeps its direction and its
    share of the step.  The returned v is not scaled.  Returns ``(x + dr, v, (dt, alpha, n_pos))``; the inputs are
    not modified."""
    dt, alpha, n_pos = state
    power = float((f * v).sum())
    if power > 0:
        v = (1 - alpha) * v + alpha * f * np.linalg.norm(v) / max(np.linalg.norm(f), 1e-30)
        n_pos += 1
        if n_pos > FIRE_N_MIN:
            dt, alpha = min(dt * FIRE_F_INC, dt_max), alpha * FIRE_F_ALPHA
    else:
        v = np.zeros_like(v)
        dt, alpha, n_pos = dt * FIRE_F_DEC, FIRE_ALPHA_START, 0
    v = v + dt * f
    dr = dt * v
    norm = np.sqrt((dr**2).sum(axis=1)).max()
    if norm > max_step:  # ase's maxstep
        dr *= max_step / norm
    return x + dr, v, (dt, alpha, n_pos)


def fire_relax(atoms, calculator: CHGNetCalculator, fmax: float = 0.1, steps: int = 500, dt: float = 0.1,
               dt_max: float = 1.0, task: PredTask = "ef", max_step: float = 0.2) -> dict:
    """Atomic-position relaxation with FIRE (Bitzek et al. 2006; the reference's default optimizer,
    dynamics.py:190-204), fixed cell, one ``fire_update`` per force evaluation.  Returns the trajectory of
    energies and the final max force."""
    v = np.zeros_like(atoms.positions)
    state = (dt, FIRE_ALPHA_START, 0)
    energies = []
    for step in range(steps):
        calculator.calculate(atoms, task=task)
        f = np.asarray(calculator.results["forces"], dtype=np.float64)
        energies.append(float(calculator.results["energy"]))
        fnorm = float(np.sqrt((f**2).sum(axis=1)).max())
        if fnorm < fmax:
            break
        atoms.positions, v, state = fire_update(atoms.positions, v, f, state, dt_max, max_step)
    return {"energies": energies, "fmax": fnorm, "steps": step + 1, "converged": fnorm < fmax}
