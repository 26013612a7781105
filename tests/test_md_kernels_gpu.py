"""-m gpu: the MD / relaxation update kernels of csrc/md.cu (chg_md_kick_drift, chg_md_kick, chg_fire_step) against
fp64 numpy restatements, called through the C ABI on synthetic data (no model).

Tolerances are derived from the operations, not fitted: u = 2^-53 is the unit roundoff of fp64, every rounding of a
result r is at most u |r|, and an n-term dot product or sum in any order (atomics, warp shuffles, BLAS) is within
gamma_n = n u / (1 - n u) times the sum of the absolute terms (Higham, Accuracy and Stability of Numerical
Algorithms, 2nd ed., Lemma 3.1 and eq. 3.5).  The kernel may contract a multiply-add into an FMA, which only removes
roundings.  Kernel and restatement round independently, so a bound on each side is doubled."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from chgnet_b200.dynamics import ATOMIC_MASSES, FS, KB, fire_update

pytestmark = pytest.mark.gpu

U = 2.0**-53
# strongly triclinic: gamma = 35 deg between a and b, c leans back over -a (139 deg) and is short in z
CELL = np.array([[6.1, 0.0, 0.0], [4.7, 3.3, 0.0], [-3.9, 2.6, 2.2]])
INV_CELL = np.ascontiguousarray(np.linalg.inv(CELL))
DT_MD = 2.0 * FS
F64 = dict(dtype=torch.float64, device="cuda")


def _gamma(k: int) -> float:
    return k * U / (1.0 - k * U)


def _lib():
    from chgnet_b200.dynamics_device import _lib

    return _lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda")


def _np(t):
    return t.cpu().numpy().copy()


def _kick_drift(x, v, f, inv_mass, dt, frac64, frac32, x_ref, max_disp2, n=None):
    return _lib().chg_md_kick_drift(_p(x), _p(v), _p(f), _p(inv_mass), x.shape[0] if n is None else n, dt,
                                    INV_CELL.ctypes.data, _p(frac64), _p(frac32), _p(x_ref), _p(max_disp2), _stream())


def _kick(v, f, inv_mass, dt, e_kin, n=None):
    return _lib().chg_md_kick(_p(v), _p(f), _p(inv_mass), v.shape[0] if n is None else n, dt, _p(e_kin), _stream())


def _fire_step(x, v, f, state, frac64, frac32, dt_max, max_step, n=None):
    return _lib().chg_fire_step(_p(x), _p(v), _p(f), x.shape[0] if n is None else n, _p(state), INV_CELL.ctypes.data,
                                _p(frac64), _p(frac32), dt_max, max_step, _stream())


def _md_inputs(n: int, seed: int):
    """Masses from H to Pu, positions spread over and beyond the cell, 600 K velocities, forces of a few eV/A."""
    rng = np.random.default_rng(seed)
    z = rng.integers(1, 95, size=n)
    z[0], z[-1] = 94, 1
    m = ATOMIC_MASSES[z - 1]
    x = rng.uniform(-0.3, 1.3, size=(n, 3)) @ CELL
    v = rng.normal(size=(n, 3)) * np.sqrt(KB * 600.0 / m)[:, None]
    f = rng.normal(scale=2.0, size=(n, 3))
    return x, v, f, 1.0 / m


def _kick_spec(v, f, inv_mass, dt):
    """v + dt/2 f/m and its bound: the kick (0.5 dt exact) carries two roundings, the sum one; one more u covers the
    second-order terms; both sides."""
    kick = 0.5 * dt * f * inv_mass[:, None]
    v_new = v + kick
    return v_new, 2.0 * (3.0 * U * np.abs(kick) + U * np.abs(v_new))


def _frac_bound(x):
    """x @ inv_cell: a 3-term dot product per component on each side."""
    return 2.0 * _gamma(3) * (np.abs(x) @ np.abs(INV_CELL))


def _exact_max_sq_norm(d):
    """max_i |d_i|^2 exactly (rational arithmetic on the candidates within rounding of the fp64 maximum)."""
    d2 = (d**2).sum(axis=1)
    cand = np.nonzero(d2 >= d2.max() * (1.0 - 16.0 * U))[0]
    return max(sum(Fraction(float(c)) ** 2 for c in d[i]) for i in cand)


def _check_max_disp2(got: float, d) -> float:
    """The kernel sums three rounded squares (three roundings): within gamma_3 of the exact value."""
    exact = _exact_max_sq_norm(d)
    err = abs(Fraction(got) - exact)
    assert err <= Fraction(_gamma(3)) * exact, (got, float(exact))
    return float(err / exact) / U


@pytest.mark.parametrize("n", [1, 255, 256, 257, 100_003])
def test_kick_drift_matches_fp64(n):
    x, v, f, im = _md_inputs(n, 100 + n)
    rng = np.random.default_rng(n)
    x_ref = x + rng.normal(scale=0.1, size=x.shape)
    xt, vt, ft, imt, xrt = (_dev(a) for a in (x, v, f, im, x_ref))
    frac64, frac32 = torch.empty(n, 3, **F64), torch.empty(n, 3, dtype=torch.float32, device="cuda")
    md2 = torch.zeros(1, **F64)
    assert _kick_drift(xt, vt, ft, imt, DT_MD, frac64, frac32, xrt, md2) == 0

    vk, xk, fk = _np(vt), _np(xt), _np(frac64)
    v_spec, bv = _kick_spec(v, f, im, DT_MD)
    assert (np.abs(vk - v_spec) <= bv).all(), np.abs(vk - v_spec).max()
    x_spec = x + DT_MD * vk  # the drift of the kernel's own velocities: one product, one sum
    bx = 2.0 * (U * np.abs(DT_MD * vk) + U * np.abs(x_spec))
    assert (np.abs(xk - x_spec) <= bx).all(), np.abs(xk - x_spec).max()
    f_spec = xk @ INV_CELL
    assert (np.abs(fk - f_spec) <= _frac_bound(xk)).all(), np.abs(fk - f_spec).max()
    assert torch.equal(frac32, frac64.float())
    ulps = _check_max_disp2(float(md2), xk - x_ref)
    print(f"n={n}: max |dv| {np.abs(vk - v_spec).max():.2e}, |dx| {np.abs(xk - x_spec).max():.2e} A, "
          f"|dfrac| {np.abs(fk - f_spec).max():.2e}, max_disp2 {ulps:.2f} u")

    # a running maximum: a smaller displacement leaves it, a larger one raises it
    before = md2.clone()
    x_now = xt.clone()
    assert _kick_drift(xt, vt, ft, imt, 0.01 * DT_MD, frac64, frac32, x_now, md2) == 0
    assert float(((xt - x_now) ** 2).sum(dim=1).max()) < 0.5 * float(before)
    assert torch.equal(md2, before)
    far = x_now - 3.0
    assert _kick_drift(xt, vt, ft, imt, 0.5 * DT_MD, frac64, frac32, far, md2) == 0
    assert float(md2) > float(before)
    _check_max_disp2(float(md2), _np(xt) - _np(far))


def test_kick_drift_optional_outputs():
    n = 257
    x, v, f, im = _md_inputs(n, 7)
    xt, vt, ft, imt = (_dev(a) for a in (x, v, f, im))
    frac64, frac32 = torch.empty(n, 3, **F64), torch.empty(n, 3, dtype=torch.float32, device="cuda")
    md2 = torch.full((1,), 7.0, **F64)
    assert _kick_drift(xt, vt, ft, imt, DT_MD, frac64, frac32, None, md2) == 0  # no reference: no displacement
    assert float(md2) == 7.0
    xs, vs = xt.clone(), vt.clone()
    assert _kick_drift(xt, vt, ft, imt, DT_MD, frac64, frac32, xs, None) == 0  # a reference but no output
    ys, ws = xs.clone(), vs.clone()
    assert _kick_drift(ys, ws, ft, imt, DT_MD, frac64.clone(), frac32.clone(), None, None) == 0
    assert torch.equal(xt, ys) and torch.equal(vt, ws)  # the optional outputs change nothing else


@pytest.mark.parametrize("n", [1, 255, 256, 257, 100_003])
def test_kick_matches_fp64_and_adds_kinetic_energy(n):
    _, v, f, im = _md_inputs(n, 200 + n)
    vt, ft, imt = _dev(v), _dev(f), _dev(im)
    e0 = 0.25
    e_kin = torch.full((1,), e0, **F64)
    assert _kick(vt, ft, imt, DT_MD, e_kin) == 0
    vk = _np(vt)
    v_spec, bv = _kick_spec(v, f, im, DT_MD)
    assert (np.abs(vk - v_spec) <= bv).all(), np.abs(vk - v_spec).max()
    want = e0 + float((0.5 / im[:, None] * vk**2).sum())
    rel = abs(float(e_kin) - want) / want
    print(f"n={n}: max |dv| {np.abs(vk - v_spec).max():.2e}, e_kin relative error {rel:.2e}")
    assert rel <= 1e-12
    # without a target the kick still happens
    vt2 = _dev(v)
    assert _kick(vt2, ft, imt, DT_MD, None) == 0
    assert torch.equal(vt2, vt)


def test_empty_and_negative_sizes():
    lib = _lib()
    n = 4
    x, v, f, im = _md_inputs(n, 3)
    xt, vt, ft, imt = (_dev(a) for a in (x, v, f, im))
    frac64, frac32 = torch.full((n, 3), -1.0, **F64), torch.full((n, 3), -1.0, dtype=torch.float32, device="cuda")
    md2, e_kin = torch.full((1,), 2.0, **F64), torch.full((1,), 3.0, **F64)
    state = torch.zeros(12, **F64)
    state[0], state[1] = 0.1, 0.1
    saved = [t.clone() for t in (xt, vt, frac64, frac32, md2, e_kin, state)]
    assert _kick_drift(xt, vt, ft, imt, DT_MD, frac64, frac32, xt.clone(), md2, n=0) == 0
    assert _kick(vt, ft, imt, DT_MD, e_kin, n=0) == 0
    assert _fire_step(xt, vt, ft, state, frac64, frac32, 1.0, 0.2, n=0) == 0
    torch.cuda.synchronize()
    for a, b in zip(saved, (xt, vt, frac64, frac32, md2, e_kin, state)):
        assert torch.equal(a, b)
    assert _kick_drift(xt, vt, ft, imt, DT_MD, frac64, frac32, None, None, n=-1) != 0
    assert b"negative size" in lib.chg_last_error()
    assert _kick(vt, ft, imt, DT_MD, None, n=-1) != 0
    assert b"negative size" in lib.chg_last_error()
    assert _fire_step(xt, vt, ft, state, frac64, frac32, 1.0, 0.2, n=-1) != 0
    assert b"negative size" in lib.chg_last_error()


# ---- chg_fire_step against chgnet_b200.dynamics.fire_update -------------------------------------------------------
DT0, DT_MAX, MAX_STEP = 0.1, 0.12, 0.2


def _springs(n: int, seed: int, stiffness):
    """Anisotropic harmonic wells: per atom and axis a stiffness from ``stiffness`` (eV/A^2), rest positions spread
    over the cell and its neighbours, start 0.6 A (rms) away from them."""
    rng = np.random.default_rng(seed)
    k = rng.choice(np.asarray(stiffness, dtype=np.float64), size=(n, 3))
    x0 = rng.uniform(-0.5, 1.5, size=(n, 3)) @ CELL
    return k, x0, x0 + 0.6 * rng.normal(size=(n, 3))


class _Fire:
    """One system on the device, stepped by chg_fire_step, forces from the springs evaluated in torch (fp64)."""

    def __init__(self, k, x0, x):
        n = x.shape[0]
        self.k, self.x0 = _dev(k), _dev(x0)
        self.x, self.v, self.f = _dev(x), torch.zeros(n, 3, **F64), torch.zeros(n, 3, **F64)
        self.frac64, self.frac32 = torch.empty(n, 3, **F64), torch.empty(n, 3, dtype=torch.float32, device="cuda")
        self.state = torch.zeros(12, **F64)
        self.state[0], self.state[1] = DT0, 0.1

    def forces(self):
        torch.mul(self.k, self.x0 - self.x, out=self.f)

    def step(self):
        assert _fire_step(self.x, self.v, self.f, self.state, self.frac64, self.frac32, DT_MAX, MAX_STEP) == 0


def _fire_bounds(x, v, f, state, dt, v_spec, x_spec, uphill):
    """Bounds on |v_kernel - v_spec| and |x_kernel - x_spec| for one step from the same (x, v, f, state).

    v' = keep v + mix f + dt f with mix = alpha |v| / |f|: the norms are 3n-term sums (gamma_3n, halved by the square
    root), mix has up to five more roundings, each product one, the two sums one each; one extra u per term covers the
    second-order terms.  x' = x + s dt v' with s = min(1, max_step / max_i |dt v'_i|): the velocity error times s dt,
    the error of s (through the norm: the velocity error, and the 3-term norm with its square root and product), and
    the two roundings of the move."""
    n = x.shape[0]
    alpha = state[1]
    c = np.abs(dt * f)
    if uphill:
        a = b = np.zeros_like(c)
    else:
        a = np.abs((1.0 - alpha) * v)
        b = np.abs(alpha * f * np.linalg.norm(v) / max(np.linalg.norm(f), 1e-30))
    bv = 2.0 * ((_gamma(3 * n) + 6.0 * U) * b + 4.0 * U * (a + b + c))
    dr = np.abs(dt * v_spec)
    norm = np.sqrt((dr**2).sum(axis=1)).max()
    d_norm = dt * np.sqrt((bv**2).sum(axis=1)).max() + 2.0 * 5.0 * U * norm
    s = min(1.0, MAX_STEP / norm) if norm > 0 else 1.0
    ds = MAX_STEP * d_norm / (norm - d_norm) ** 2 + 2.0 * U if norm + d_norm > MAX_STEP else 0.0
    bx = s * dt * bv + ds * dr + 2.0 * (3.0 * U * s * dr + U * np.abs(x_spec))
    return bv, bx


@pytest.mark.parametrize("n", [7, 1000, 70_001])
def test_fire_step_follows_fire_update_step_by_step(n):
    """80 steps of chg_fire_step; before each one the device state is copied and fire_update takes the same step from
    it.  The trajectory must visit every branch of FIRE, and the step limit must scale the whole update."""
    dev = _Fire(*_springs(n, 300 + n, (0.5, 2.0, 8.0, 30.0)))
    seen = dict(first_uphill=False, grow_past_n_min=False, reach_dt_max=False, alpha_decay=False, reset=False,
                clamp=False)
    skipped, worst = [], dict(v=0.0, x=0.0, frac=0.0, f2=0.0)
    for step in range(80):
        dev.forces()
        x, v, f, st = (_np(t) for t in (dev.x, dev.v, dev.f, dev.state))
        dev.step()
        xk, vk, stk, fk = _np(dev.x), _np(dev.v), _np(dev.state), _np(dev.frac64)

        assert (stk[3:8] == 0.0).all(), stk  # the scratch slots are clean for the next step
        ff = (f**2).sum(axis=1).max()
        worst["f2"] = max(worst["f2"], abs(stk[11] - ff) / ff)
        assert abs(stk[11] - ff) <= 2.0 * _gamma(3) * ff
        assert (stk[8:11] == stk[0:3]).all()
        assert torch.equal(dev.frac32, dev.frac64.float())
        assert (np.abs(fk - xk @ INV_CELL) <= _frac_bound(xk)).all()
        worst["frac"] = max(worst["frac"], np.abs(fk - xk @ INV_CELL).max())

        power = float((f * v).sum())
        if abs(power) <= 2.0 * _gamma(3 * n) * float(np.abs(f * v).sum()) and power != 0.0:
            skipped.append(step)  # the sign of f.v is within rounding: either branch is right
            continue
        x_spec, v_spec, (dt, alpha, n_pos) = fire_update(x, v, f, (st[0], st[1], int(st[2])), DT_MAX, MAX_STEP)
        assert (stk[0], stk[1], stk[2]) == (dt, alpha, float(n_pos)), (step, stk[:3], (dt, alpha, n_pos))

        uphill = not power > 0
        seen["first_uphill"] |= step == 0 and uphill and dt == DT0 * 0.5
        seen["grow_past_n_min"] |= n_pos > 5 and dt > st[0]
        seen["reach_dt_max"] |= st[0] < DT_MAX and dt == DT_MAX
        seen["alpha_decay"] |= alpha < st[1]
        seen["reset"] |= step > 0 and uphill and st[2] > 0
        unclamped = np.sqrt(((dt * v_spec) ** 2).sum(axis=1))
        if unclamped.max() > MAX_STEP:
            s = MAX_STEP / unclamped.max()
            moved = np.sqrt(((xk - x) ** 2).sum(axis=1))
            i = int(np.argmin(moved))
            if s < 0.9:
                seen["clamp"] = True
                # the step limit scales every atom, not only the ones beyond max_step
                assert moved[i] < unclamped[i] * (1.0 - 0.5 * (1.0 - s)), (step, i, moved[i], unclamped[i], s)

        bv, bx = _fire_bounds(x, v, f, st, dt, v_spec, x_spec, uphill)
        assert (np.abs(vk - v_spec) <= bv).all(), (step, np.abs(vk - v_spec).max())
        assert (np.abs(xk - x_spec) <= bx).all(), (step, np.abs(xk - x_spec).max())
        worst["v"] = max(worst["v"], np.abs(vk - v_spec).max())
        worst["x"] = max(worst["x"], np.abs(xk - x_spec).max())
    print(f"n={n}: max |dv| {worst['v']:.2e}, |dx| {worst['x']:.2e} A, |dfrac| {worst['frac']:.2e}, "
          f"max|f_i|^2 relative {worst['f2']:.2e}; steps with f.v within rounding of 0 (branch not compared): {skipped}")
    assert seen == dict.fromkeys(seen, True), seen
    assert len(skipped) <= 2


def test_fire_step_free_run_matches_fire_update():
    """40 steps on each side from the same start, each following its own trajectory (soft springs: stable)."""
    k, x0, x = _springs(1000, 77, (0.5, 1.0, 2.0))
    dev = _Fire(k, x0, x)
    v, state = np.zeros_like(x), (DT0, 0.1, 0)
    for _ in range(40):
        dev.forces()
        dev.step()
        x, v, state = fire_update(x, v, k * (x0 - x), state, DT_MAX, MAX_STEP)
    dx = np.abs(_np(dev.x) - x).max()
    st = _np(dev.state)
    print(f"40 free steps: max |x_kernel - x_spec| {dx:.2e} A, state {st[:3]} vs {state}")
    assert dx <= 1e-10
    assert (st[0], st[1], st[2]) == (state[0], state[1], float(state[2]))
