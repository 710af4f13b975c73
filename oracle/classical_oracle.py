"""CPU restatement of the classical predictors' arithmetic -- TEST INFRASTRUCTURE.

PARITY UNPINNED vs upstream: the arithmetic of the reference's classical predictors lives in
third-party packages that are neither vendored in /root/reference nor installable here, and the
reference holds no tests for them:
  * socialforce (svenkreiss/socialforce, pre-PyTorch v0.1.x API, unpinned) -- call sites
    trajnetbaselines/classical/socialforce.py:6-8,89-93
  * pykalman (unpinned, setup.py:25)  -- call sites classical/kalman.py:40-55
  * rvo2 (sybrenstuvel/Python-RVO2 over snape/RVO2 v2.0.x) -- oracle/orca_oracle.c
The functions below restate the published algorithms those call sites exercise (Helbing &
Molnar 1995 as implemented by socialforce v0.1.x; Shumway-Stoffer EM / RTS smoother as
implemented by pykalman's default `em`), float64 like upstream, and follow the reference's
own adapter code for everything around them (initial state, sampling quirks).
constant_velocity (classical/constant_velocity.py:4-20) is fully in-repo and exact.
"""
import numpy as np


# ----------------------------------------------------------------------------------------
# social force: socialforce.Simulator.step (v0.1.x), as driven by classical/socialforce.py:89-95
# ----------------------------------------------------------------------------------------
def _sf_b(r_ab, speeds, e, delta_t):
    """Semi-minor axis of the elliptical potential.  r_ab [N,N,2], speeds [N], e [N,2]."""
    speeds_b = speeds[None, :]                                    # indexed by b
    e_b = e[None, :, :]
    in_sqrt = (np.linalg.norm(r_ab, axis=-1) +
               np.linalg.norm(r_ab - delta_t * speeds_b[..., None] * e_b, axis=-1)) ** 2 - \
              (delta_t * speeds_b) ** 2
    np.fill_diagonal(in_sqrt, 0.0)
    return 0.5 * np.sqrt(in_sqrt)


def _sf_value(r_ab, speeds, e, delta_t, v0, sigma):
    return v0 * np.exp(-_sf_b(r_ab, speeds, e, delta_t) / sigma)


def sf_step(state, initial_speeds, max_speeds, delta_t, v0, sigma, fd_delta=1e-3,
            twophi=200.0, out_of_view_factor=0.5, counters=None):
    """One Simulator.step().  state [N,7] float64 (x,y,vx,vy,dx,dy,tau), updated in place.
    counters: None, or a dict that gets SF_COUNTERS added to it (pairs a != b weighted out of view; pedestrians
    whose speed is clipped to max_speeds)."""
    pos = state[:, 0:2]
    vel = state[:, 2:4]
    dest = state[:, 4:6]
    tau = state[:, 6:7]
    dvec = dest - pos
    e = dvec / np.linalg.norm(dvec, axis=-1, keepdims=True)       # desired directions
    F0 = 1.0 / tau * (initial_speeds[:, None] * e - vel)
    # pedestrian-pedestrian repulsion: f_ab = -grad_{r_ab} V, forward finite differences
    speeds = np.linalg.norm(vel, axis=-1)
    r_ab = pos[:, None, :] - pos[None, :, :]
    dx = np.array([[[fd_delta, 0.0]]])
    dy = np.array([[[0.0, fd_delta]]])
    v = _sf_value(r_ab, speeds, e, delta_t, v0, sigma)
    dvdx = (_sf_value(r_ab + dx, speeds, e, delta_t, v0, sigma) - v) / fd_delta
    dvdy = (_sf_value(r_ab + dy, speeds, e, delta_t, v0, sigma) - v) / fd_delta
    np.fill_diagonal(dvdx, 0.0)
    np.fill_diagonal(dvdy, 0.0)
    f_ab = -1.0 * np.stack((dvdx, dvdy), axis=-1)
    # field of view weight w(e, -f_ab)
    cosphi = np.cos(twophi / 2.0 / 180.0 * np.pi)
    f = -f_ab
    in_sight = np.einsum('aj,abj->ab', e, f) > np.linalg.norm(f, axis=-1) * cosphi
    w = out_of_view_factor * np.ones_like(in_sight, dtype=np.float64)
    w[in_sight] = 1.0
    np.fill_diagonal(w, 0.0)
    # sum over b = 0 .. N-1 in index order, then F0 + sum: one rounding order, the one the CUDA kernel uses
    wf = w[..., None] * f_ab
    total = np.zeros_like(F0)
    for b in range(len(state)):
        total += wf[:, b]
    F = F0 + total
    wv = vel + delta_t * F
    desired = np.linalg.norm(wv, axis=-1)
    with np.errstate(divide='ignore', invalid='ignore'):
        q = max_speeds / desired
        factor = np.minimum(1.0, q)
    if counters is not None:
        off_diagonal = ~np.eye(len(state), dtype=bool)
        counters['out_of_view'] = counters.get('out_of_view', 0) + int((~in_sight & off_diagonal).sum())
        counters['speed_clip'] = counters.get('speed_clip', 0) + int((q < 1.0).sum())
    v_new = wv * factor[:, None]
    state[:, 0:2] = pos + v_new * delta_t
    state[:, 2:4] = v_new
    return state


SF_COUNTERS = ('out_of_view', 'speed_clip')


def sf_simulate(initial_state, delta_t=0.05, tau=0.5, v0=2.1, sigma=0.3, n_steps=96, sample_every=8,
                counters=None):
    """classical/socialforce.py:89-95: n_steps x step(), keep the states whose index % 8 == 0
    (i.e. after sim steps 1, 9, 17, ...).  initial_state [N,6] -> [n_samples, N, 2].
    counters: None, or a dict that sums sf_step's counters over the steps."""
    state = np.concatenate([np.asarray(initial_state, dtype=np.float64),
                            np.full((len(initial_state), 1), tau)], axis=1)
    initial_speeds = np.linalg.norm(state[:, 2:4], axis=-1)
    max_speeds = 1.3 * initial_speeds
    out = []
    with np.errstate(divide='ignore', invalid='ignore'):
        for k in range(n_steps):
            sf_step(state, initial_speeds, max_speeds, delta_t, v0, sigma, counters=counters)
            if k % sample_every == 0:
                out.append(state[:, 0:2].copy())
    return np.stack(out)


# ----------------------------------------------------------------------------------------
# initial state shared by socialforce / orca adapters (classical/socialforce.py:15-72)
# ----------------------------------------------------------------------------------------
def adapter_initial_states(xy_obs, pred_length=12):
    """xy_obs [obs_len, N, 2] float64 with NaN for absent frames; returns rows for peds present at
    the last observed frame: (x, y, vx, vy, dx, dy), speed, keep-mask."""
    T, N, _ = xy_obs.shape
    rows, speeds, keep = [], [], []
    for p in range(N):
        present = ~np.isnan(xy_obs[:, p, 0])
        if not present[-1]:
            keep.append(False)
            continue
        keep.append(True)
        path = xy_obs[present, p]
        n = len(path)
        curr = path[-1]
        if n >= 4:
            stride, prev = 3, path[-4]
        else:
            stride, prev = n - 1, path[0]
        if stride == 0:
            vx = vy = speed = 0.0
        else:
            diff = curr - prev
            theta = np.arctan2(diff[1], diff[0])
            speed = np.linalg.norm(diff) / (stride * 0.4)
            vx, vy = speed * np.cos(theta), speed * np.sin(theta)
        if n == 1:
            d = curr
        else:   # interp1d(fill_value='extrapolate') at time n-1+pred_length: linear on the last segment
            d = path[-1] + (path[-1] - path[-2]) * pred_length
        rows.append([curr[0], curr[1], vx, vy, d[0], d[1]])
        speeds.append(speed)
    return np.array(rows, dtype=np.float64).reshape(-1, 6), np.array(speeds), np.array(keep)


def constant_velocity(xy_obs, n_predict=12):
    """classical/constant_velocity.py:4-20."""
    curr = xy_obs[-1]
    vel = xy_obs[-1] - xy_obs[-2]
    return curr[None] + np.arange(1, n_predict + 1)[:, None, None] * vel[None]


# ----------------------------------------------------------------------------------------
# Kalman: pykalman.KalmanFilter(em -> smooth -> expected rollout), classical/kalman.py:31-60
# ----------------------------------------------------------------------------------------
def _kf_filter(A, C, Q, R, mu0, S0, Z):
    T = len(Z)
    n = A.shape[0]
    pm = np.zeros((T, n)); pc = np.zeros((T, n, n))       # predicted
    fm = np.zeros((T, n)); fc = np.zeros((T, n, n))       # filtered
    K = np.zeros((T, n, C.shape[0]))
    for t in range(T):
        if t == 0:
            pm[t], pc[t] = mu0, S0
        else:
            pm[t] = A @ fm[t - 1]
            pc[t] = A @ fc[t - 1] @ A.T + Q
        S = C @ pc[t] @ C.T + R
        K[t] = pc[t] @ C.T @ np.linalg.pinv(S)
        fm[t] = pm[t] + K[t] @ (Z[t] - C @ pm[t])
        fc[t] = pc[t] - K[t] @ C @ pc[t]
    return pm, pc, K, fm, fc


def _kf_smooth(A, pm, pc, fm, fc):
    T, n = fm.shape
    sm = np.zeros((T, n)); sc = np.zeros((T, n, n)); G = np.zeros((T - 1, n, n))
    sm[-1], sc[-1] = fm[-1], fc[-1]
    for t in reversed(range(T - 1)):
        G[t] = fc[t] @ A.T @ np.linalg.pinv(pc[t + 1])
        sm[t] = fm[t] + G[t] @ (sm[t + 1] - pm[t + 1])
        sc[t] = fc[t] + G[t] @ (sc[t + 1] - pc[t + 1]) @ G[t].T
    return sm, sc, G


def kalman_predict_track(obs, n_predict=12, n_iter=10):
    """EM (transition_covariance, observation_covariance, initial_state_mean, initial_state_covariance;
    pykalman's default em_vars) -> RTS smoother -> expected observation rollout C A^k x_last.

    obs [T, 2].  The reference averages 5 noisy `kf.sample` draws from the unseeded global numpy
    RNG (kalman.py:53-60); their expectation is what is restated here."""
    Z = np.asarray(obs, dtype=np.float64)
    T = len(Z)
    A = np.array([[1, 1, 0, 0], [0, 1, 0, 0], [0, 0, 1, 1], [0, 0, 0, 1]], dtype=np.float64)
    C = np.array([[1, 0, 0, 0], [0, 0, 1, 0]], dtype=np.float64)
    Q = 1e-5 * np.eye(4)
    R = 0.05 ** 2 * np.eye(2)
    mu0 = np.array([Z[0, 0], 0, Z[0, 1], 0], dtype=np.float64)
    S0 = np.eye(4)
    for _ in range(n_iter):
        pm, pc, K, fm, fc = _kf_filter(A, C, Q, R, mu0, S0, Z)
        sm, sc, G = _kf_smooth(A, pm, pc, fm, fc)
        # pairwise covariances Cov(x_t, x_{t-1} | Z)
        pair = np.zeros((T, 4, 4))
        for t in range(1, T):
            pair[t] = sc[t] @ G[t - 1].T
        # M-step
        Rn = np.zeros((2, 2))
        for t in range(T):
            err = Z[t] - C @ sm[t]
            Rn += np.outer(err, err) + C @ sc[t] @ C.T
        R = Rn / T
        Qn = np.zeros((4, 4))
        for t in range(T - 1):
            err = sm[t + 1] - A @ sm[t]
            Vt1t_A = pair[t + 1] @ A.T
            Qn += np.outer(err, err) + A @ sc[t] @ A.T + sc[t + 1] - Vt1t_A - Vt1t_A.T
        Q = Qn / (T - 1)
        mu0 = sm[0].copy()
        S0 = sc[0].copy()
    pm, pc, K, fm, fc = _kf_filter(A, C, Q, R, mu0, S0, Z)
    sm, sc, G = _kf_smooth(A, pm, pc, fm, fc)
    x = sm[-1].copy()
    out = np.zeros((n_predict, 2))
    for k in range(n_predict):
        x = A @ x
        out[k] = C @ x
    return out
