"""Complex-step restatement of the social-force rollout -- TEST INFRASTRUCTURE.

oracle/classical_oracle.sf_step with complex128 state: one swept parameter (tau, v0 or sigma) carries an imaginary
step i h, so imag(f) / h is df/dtheta to float64 precision, with no subtraction and no step-size trade-off (Squire &
Trapp 1998).  It checks the forward-mode duals of tb2_sf_sweep_grad by a method that shares nothing with them.

Differences from sf_step, all forced by complex arithmetic: |v| is sqrt(x*x + y*y) (np.linalg.norm would return the
modulus), and the comparisons -- the field-of-view test and numpy.minimum(1, q) -- act on the real part, so each takes
the branch the real rollout takes and the derivative is that branch's.
"""
import numpy as np

H = 1e-30                                    # imaginary step: far below any rounding of the real part


def _norm(v):
    return np.sqrt(v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1])


def _sf_value(r_ab, speeds, e, delta_t, v0, sigma):
    speeds_b = speeds[None, :]
    e_b = e[None, :, :]
    in_sqrt = (_norm(r_ab) + _norm(r_ab - delta_t * speeds_b[..., None] * e_b)) ** 2 - (delta_t * speeds_b) ** 2
    np.fill_diagonal(in_sqrt, 0.0)
    return v0 * np.exp(-(0.5 * np.sqrt(in_sqrt)) / sigma)


def _sf_step(state, initial_speeds, max_speeds, delta_t, tau, v0, sigma, fd_delta=1e-3, twophi=200.0,
             out_of_view_factor=0.5):
    pos, vel, dest = state[:, 0:2], state[:, 2:4], state[:, 4:6]
    dvec = dest - pos
    e = dvec / _norm(dvec)[:, None]
    F0 = 1.0 / tau * (initial_speeds[:, None] * e - vel)
    speeds = _norm(vel)
    r_ab = pos[:, None, :] - pos[None, :, :]
    v = _sf_value(r_ab, speeds, e, delta_t, v0, sigma)
    dvdx = (_sf_value(r_ab + np.array([[[fd_delta, 0.0]]]), speeds, e, delta_t, v0, sigma) - v) / fd_delta
    dvdy = (_sf_value(r_ab + np.array([[[0.0, fd_delta]]]), speeds, e, delta_t, v0, sigma) - v) / fd_delta
    np.fill_diagonal(dvdx, 0.0)
    np.fill_diagonal(dvdy, 0.0)
    f_ab = -1.0 * np.stack((dvdx, dvdy), axis=-1)
    cosphi = np.cos(twophi / 2.0 / 180.0 * np.pi)
    f = -f_ab
    in_sight = np.einsum('aj,abj->ab', e, f).real > (_norm(f) * cosphi).real
    w = np.where(in_sight, 1.0, out_of_view_factor)
    np.fill_diagonal(w, 0.0)
    wf = w[..., None] * f_ab
    total = np.zeros_like(F0)
    for b in range(len(state)):
        total += wf[:, b]
    wv = vel + delta_t * (F0 + total)
    q = max_speeds / _norm(wv)
    factor = np.where(np.isnan(q.real) | (q.real < 1.0), q, 1.0)          # numpy.minimum(1, q) on the real part
    v_new = wv * factor[:, None]
    state[:, 0:2] = pos + v_new * delta_t
    state[:, 2:4] = v_new


def sf_simulate_cs(initial_state, tau, v0, sigma, which, delta_t=0.05, n_steps=96, sample_every=8):
    """sf_simulate with parameter `which` (0 tau, 1 v0, 2 sigma) stepped by i H -> complex positions [n_samples, N, 2]:
    .real the rollout, .imag / H its derivative with respect to that parameter."""
    theta = [complex(tau), complex(v0), complex(sigma)]
    theta[which] += 1j * H
    st = np.asarray(initial_state, dtype=np.float64).astype(np.complex128)
    initial_speeds = np.sqrt(st[:, 2].real ** 2 + st[:, 3].real ** 2)
    max_speeds = 1.3 * initial_speeds
    out = []
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        for k in range(n_steps):
            _sf_step(st, initial_speeds, max_speeds, delta_t, *theta)
            if k % sample_every == 0:
                out.append(st[:, 0:2].copy())
    return np.stack(out)


def score_cs(truth, primary):
    """(ADE, FDE) of a complex primary track [n_samples, 2] against real truth: distances summed in sample order."""
    e = truth - primary
    d = np.sqrt(e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1])
    s = 0.0
    for v in d:
        s = s + v
    return s / len(d), d[-1]


def score_grad(initial_state, truth, tau, v0, sigma, **kw):
    """(ade, fde, dade [3], dfde [3]) of the scene's primary (row 0) by three complex-step rollouts."""
    dade, dfde = np.empty(3), np.empty(3)
    for which in range(3):
        with np.errstate(invalid='ignore'):
            a, f = score_cs(truth, sf_simulate_cs(initial_state, tau, v0, sigma, which, **kw)[:, 0])
        dade[which], dfde[which] = a.imag / H, f.imag / H
    return a.real, f.real, dade, dfde
