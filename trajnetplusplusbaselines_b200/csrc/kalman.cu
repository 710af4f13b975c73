// Kalman predictor, float64, one code for the host and the device.
//
// Replaces the pykalman calls of trajnetbaselines/classical/kalman.py:40-60:
//   KalmanFilter(A = constant-velocity 4x4, C = 2x4, Q = 1e-5 I, R = 0.05^2 I, mu0 = (x0,0,y0,0))
//   .em(obs)            default em_vars: Q, R, mu0, Sigma0; 10 iterations
//   .smooth(obs)        RTS smoother, last smoothed mean = initial_state of the rollout
//   mean of 5 x .sample(n_predict + 1)   -> here: the expectation C A^k x_last plus the fitted
//                       Q, R so the caller can add the reference's sampled noise.
// pykalman is not vendored (parity unpinned, see oracle/classical_oracle.py); the EM follows
// Shumway & Stoffer as pykalman documents it.
//
// Two entry points run the same __host__ __device__ EM / smoother / rollout:
//   tb2_kalman_predict         host C++ (BASELINE configs[0] is CPU-only), tracks fanned out over host threads;
//   tb2_kalman_predict_device  one CUDA thread per track, the track's T-length arrays interleaved over the tracks in a
//                              caller-owned workspace; optionally adds the noise of the reference's sampled rollouts.
// The file is compiled with -fmad=false and the host side by g++ for baseline x86-64 (no FMA): both sides run the
// same operations in the same order, so the device's expectation, Q, R and last state equal the host's bit for bit.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <thread>
#include <vector>

#include "common.cuh"

#define TB2_HD __host__ __device__ inline
#ifdef __CUDA_ARCH__
#define TB2_UNROLL _Pragma("unroll")
#else
#define TB2_UNROLL
#endif

namespace {

struct M4 { double a[4][4]; };
struct V4 { double a[4]; };

TB2_HD M4 zero4() { M4 r; for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) r.a[i][j] = 0.0; return r; }
TB2_HD M4 eye4(double s) { M4 r = zero4(); for (int i = 0; i < 4; ++i) r.a[i][i] = s; return r; }
TB2_HD M4 mul(const M4& x, const M4& y) {
    M4 r = zero4();
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) { double s = 0; for (int k = 0; k < 4; ++k) s += x.a[i][k] * y.a[k][j]; r.a[i][j] = s; }
    return r;
}
TB2_HD M4 tr(const M4& x) { M4 r; for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) r.a[i][j] = x.a[j][i]; return r; }
TB2_HD M4 add(const M4& x, const M4& y) { M4 r; for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) r.a[i][j] = x.a[i][j] + y.a[i][j]; return r; }
TB2_HD M4 sub(const M4& x, const M4& y) { M4 r; for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) r.a[i][j] = x.a[i][j] - y.a[i][j]; return r; }
TB2_HD V4 mulv(const M4& x, const V4& v) { V4 r; for (int i = 0; i < 4; ++i) { double s = 0; for (int k = 0; k < 4; ++k) s += x.a[i][k] * v.a[k]; r.a[i] = s; } return r; }
TB2_HD M4 outer(const V4& u, const V4& v) { M4 r; for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) r.a[i][j] = u.a[i] * v.a[j]; return r; }

TB2_HD M4 transition() {
    M4 A = eye4(1.0);
    A.a[0][1] = 1.0;
    A.a[2][3] = 1.0;
    return A;
}

// inverse of a 4x4 by Gauss-Jordan with partial pivoting (covariances here are SPD).  The row swap walks the rows with
// compile-time indices, so on the device the working matrix stays in registers.
TB2_HD bool inv4(const M4& m, M4& out) {
    double w[4][8];
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) { w[i][j] = m.a[i][j]; w[i][j + 4] = (i == j) ? 1.0 : 0.0; }
TB2_UNROLL
    for (int c = 0; c < 4; ++c) {
        int piv = c;
        double best = w[c][c];
TB2_UNROLL
        for (int r = c + 1; r < 4; ++r) if (fabs(w[r][c]) > fabs(best)) { piv = r; best = w[r][c]; }
        if (fabs(best) < 1e-300) return false;
TB2_UNROLL
        for (int r = c + 1; r < 4; ++r)
            if (r == piv)
TB2_UNROLL
                for (int j = 0; j < 8; ++j) { const double t = w[r][j]; w[r][j] = w[c][j]; w[c][j] = t; }
        const double d = w[c][c];
TB2_UNROLL
        for (int j = 0; j < 8; ++j) w[c][j] /= d;
TB2_UNROLL
        for (int r = 0; r < 4; ++r) if (r != c) { const double f = w[r][c]; if (f != 0.0) for (int j = 0; j < 8; ++j) w[r][j] -= f * w[c][j]; }
    }
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) out.a[i][j] = w[i][j + 4];
    return true;
}

// The T-length arrays of one track (predicted / filtered / smoothed means and covariances, smoother gains): field f of
// step k lives at base[(k * kFields + f) * stride].  Host: the track's own buffer, stride 1.  Device: the workspace as
// [k][field][track], base = workspace + track, stride = n_tracks, so the loads of a warp's 32 tracks coalesce.
constexpr int kPM = 0, kFM = 4, kSM = 8, kPC = 12, kFC = 28, kSC = 44, kG = 60, kFields = 76;

struct TrackView {
    double* base;
    int64_t stride;
    TB2_HD double& at(int k, int f) const { return base[((int64_t)k * kFields + f) * stride]; }
    TB2_HD V4 v(int k, int f) const { V4 r; for (int i = 0; i < 4; ++i) r.a[i] = at(k, f + i); return r; }
    TB2_HD M4 m(int k, int f) const {
        M4 r;
        for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) r.a[i][j] = at(k, f + 4 * i + j);
        return r;
    }
    TB2_HD void put(int k, int f, const V4& x) const { for (int i = 0; i < 4; ++i) at(k, f + i) = x.a[i]; }
    TB2_HD void put(int k, int f, const M4& x) const { for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) at(k, f + 4 * i + j) = x.a[i][j]; }
};

// observation model C = [[1,0,0,0],[0,0,1,0]] is applied by index (state 0 -> x, state 2 -> y)
TB2_HD void filter(const M4& A, const M4& At, const M4& Q, const double R[2][2], const V4& mu0, const M4& S0,
                   const double* Z, int T, const TrackView& t) {
    V4 fm;
    M4 fc;
    for (int k = 0; k < T; ++k) {
        V4 pm;
        M4 P;
        if (k == 0) { pm = mu0; P = S0; }
        else { pm = mulv(A, fm); P = add(mul(mul(A, fc), At), Q); }
        // S = C P C^T + R (2x2), K = P C^T S^-1 (4x2)
        const double s00 = P.a[0][0] + R[0][0], s01 = P.a[0][2] + R[0][1];
        const double s10 = P.a[2][0] + R[1][0], s11 = P.a[2][2] + R[1][1];
        const double det = s00 * s11 - s01 * s10;
        const double i00 = s11 / det, i01 = -s01 / det, i10 = -s10 / det, i11 = s00 / det;
        double K[4][2];
        for (int i = 0; i < 4; ++i) {
            K[i][0] = P.a[i][0] * i00 + P.a[i][2] * i10;
            K[i][1] = P.a[i][0] * i01 + P.a[i][2] * i11;
        }
        const double e0 = Z[2 * k] - pm.a[0], e1 = Z[2 * k + 1] - pm.a[2];
        for (int i = 0; i < 4; ++i) fm.a[i] = pm.a[i] + K[i][0] * e0 + K[i][1] * e1;
        // fc = P - K C P
        for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j)
            fc.a[i][j] = P.a[i][j] - (K[i][0] * P.a[0][j] + K[i][1] * P.a[2][j]);
        t.put(k, kPM, pm); t.put(k, kPC, P);
        t.put(k, kFM, fm); t.put(k, kFC, fc);
    }
}

TB2_HD bool smooth(const M4& At, int T, const TrackView& t) {
    V4 sm = t.v(T - 1, kFM);                 // smoothed mean / covariance of step k + 1 while step k is computed
    M4 sc = t.m(T - 1, kFC);
    t.put(T - 1, kSM, sm);
    t.put(T - 1, kSC, sc);
    for (int k = T - 2; k >= 0; --k) {
        const M4 pc1 = t.m(k + 1, kPC);
        M4 pinv;
        if (!inv4(pc1, pinv)) return false;
        const M4 fc = t.m(k, kFC);
        const M4 G = mul(mul(fc, At), pinv);
        const V4 pm1 = t.v(k + 1, kPM), fm = t.v(k, kFM);
        V4 d;
        for (int i = 0; i < 4; ++i) d.a[i] = sm.a[i] - pm1.a[i];
        const V4 gd = mulv(G, d);
        for (int i = 0; i < 4; ++i) sm.a[i] = fm.a[i] + gd.a[i];
        sc = add(fc, mul(mul(G, sub(sc, pc1)), tr(G)));
        t.put(k, kG, G);
        t.put(k, kSM, sm);
        t.put(k, kSC, sc);
    }
    return true;
}

// One track: EM (Q, R, mu0, Sigma0) and the smoother.  Z: the track's T >= 2 observations [T, 2].  Returns false on a
// singular predicted covariance; on success Q, R and the last smoothed state `last` are set.
TB2_HD bool kalman_fit(const double* Z, int T, int em_iterations, const TrackView& t, M4& Q, double R[2][2], V4& last) {
    const M4 A = transition();
    const M4 At = tr(A);
    Q = eye4(1e-5);
    R[0][0] = 0.05 * 0.05; R[0][1] = 0.0; R[1][0] = 0.0; R[1][1] = 0.05 * 0.05;
    V4 mu0 = {{Z[0], 0.0, Z[1], 0.0}};
    M4 S0 = eye4(1.0);
    for (int it = 0; it < em_iterations; ++it) {
        filter(A, At, Q, R, mu0, S0, Z, T, t);
        if (!smooth(At, T, t)) return false;
        // M-step (pykalman _em_observation_covariance / _em_transition_covariance / initial state)
        double Rn[2][2] = {{0, 0}, {0, 0}};
        for (int k = 0; k < T; ++k) {
            const V4 sm = t.v(k, kSM);
            const M4 sc = t.m(k, kSC);
            const double e0 = Z[2 * k] - sm.a[0], e1 = Z[2 * k + 1] - sm.a[2];
            Rn[0][0] += e0 * e0 + sc.a[0][0];
            Rn[0][1] += e0 * e1 + sc.a[0][2];
            Rn[1][0] += e1 * e0 + sc.a[2][0];
            Rn[1][1] += e1 * e1 + sc.a[2][2];
        }
        for (int i = 0; i < 2; ++i) for (int j = 0; j < 2; ++j) R[i][j] = Rn[i][j] / T;
        M4 Qn = zero4();
        V4 sm0 = t.v(0, kSM);
        M4 sc0 = t.m(0, kSC);
        mu0 = sm0;
        S0 = sc0;
        for (int k = 0; k < T - 1; ++k) {
            const V4 sm1 = t.v(k + 1, kSM);
            const M4 sc1 = t.m(k + 1, kSC);
            const V4 ax = mulv(A, sm0);
            V4 err;
            for (int i = 0; i < 4; ++i) err.a[i] = sm1.a[i] - ax.a[i];
            const M4 pair = mul(sc1, tr(t.m(k, kG)));      // Cov(x_{k+1}, x_k | Z)
            const M4 pa = mul(pair, At);
            M4 term = add(outer(err, err), mul(mul(A, sc0), At));
            term = add(term, sc1);
            term = sub(term, pa);
            term = sub(term, tr(pa));
            Qn = add(Qn, term);
            sm0 = sm1;
            sc0 = sc1;
        }
        for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) Q.a[i][j] = Qn.a[i][j] / (T - 1);
    }
    filter(A, At, Q, R, mu0, S0, Z, T, t);
    if (!smooth(At, T, t)) return false;
    last = t.v(T - 1, kSM);
    return true;
}

// Lower factor L with L L^T = (S + S^T) / 2 of a positive-semidefinite N x N matrix, possibly singular (a fitted Q of a
// short track is close to rank-deficient; the M-step's sums leave it symmetric only to rounding): Cholesky with a
// zero-pivot guard.  A pivot not above 1e-12 x the largest diagonal entry (zero, or negative by rounding) zeroes its
// column, which is what the exact factor of a singular PSD matrix holds there.
template <int N>
TB2_HD void chol_psd(const double* S, double* L) {
    double dmax = 0.0;
    for (int i = 0; i < N; ++i) dmax = fmax(dmax, S[i * N + i]);
    const double tol = 1e-12 * dmax;
    for (int i = 0; i < N * N; ++i) L[i] = 0.0;
    for (int j = 0; j < N; ++j) {
        double d = S[j * N + j];
        for (int k = 0; k < j; ++k) d -= L[j * N + k] * L[j * N + k];
        if (!(d > tol)) continue;
        const double ljj = sqrt(d);
        L[j * N + j] = ljj;
        for (int i = j + 1; i < N; ++i) {
            double s = 0.5 * (S[i * N + j] + S[j * N + i]);
            for (int k = 0; k < j; ++k) s -= L[i * N + k] * L[j * N + k];
            L[i * N + j] = s / ljj;
        }
    }
}

// Rollout from the last smoothed state: pred[k] = C A^(k+1) x_last (k = 0 .. n_predict - 1).  With eps (device only),
// the noise of the mean of n_samples sampled rollouts is added: the noise enters linearly and the rollouts are i.i.d.,
// so that mean is the expectation plus ONE deviation driven by Q / n and R / n,
//   dx_k = A dx_{k-1} + LQ e_k[0:4] / sqrt(n),  pred[k] += (dx_k[0], dx_k[2]) + LR e_k[4:6] / sqrt(n),  dx_0 = 0,
// with LQ, LR the chol_psd factors of Q and R and e [n_predict, 6] standard normals.  z_0 is never formed (the
// reference drops it).  The expectation is computed by the same operations with or without noise.
TB2_HD void rollout(V4 x, int n_predict, double* pred, const double* eps, int n_samples, const M4& Q, const double R[2][2]) {
    const M4 A = transition();
    double LQ[16], LR[4], scale = 0.0;
    V4 dx = {{0.0, 0.0, 0.0, 0.0}};
    if (eps) {
        chol_psd<4>(&Q.a[0][0], LQ);
        chol_psd<2>(&R[0][0], LR);
        scale = 1.0 / sqrt((double)n_samples);
    }
    for (int k = 0; k < n_predict; ++k) {
        x = mulv(A, x);
        double px = x.a[0], py = x.a[2];
        if (eps) {
            const double* e = eps + 6 * k;
            dx = mulv(A, dx);
            for (int i = 0; i < 4; ++i) {
                double w = 0.0;
                for (int j = 0; j <= i; ++j) w += LQ[i * 4 + j] * e[j];
                dx.a[i] += scale * w;
            }
            const double v0 = LR[0] * e[4], v1 = LR[2] * e[4] + LR[3] * e[5];
            px += dx.a[0] + scale * v0;
            py += dx.a[2] + scale * v1;
        }
        pred[2 * k + 0] = px;
        pred[2 * k + 1] = py;
    }
}

TB2_HD void write_fit(int64_t i, const M4& Q, const double R[2][2], const V4& x, double* q_out, double* r_out,
                      double* last_state_out) {
    if (last_state_out) for (int j = 0; j < 4; ++j) last_state_out[i * 4 + j] = x.a[j];
    if (q_out) for (int a = 0; a < 4; ++a) for (int b = 0; b < 4; ++b) q_out[i * 16 + a * 4 + b] = Q.a[a][b];
    if (r_out) for (int a = 0; a < 2; ++a) for (int b = 0; b < 2; ++b) r_out[i * 4 + a * 2 + b] = R[a][b];
}

// One track on the host.  Returns nullptr or a static error message; tracks are independent, so the caller may run them
// on several host threads (results do not depend on the thread count).  `buf` is the calling thread's scratch.
const char* kalman_track(int tr_i, const double* obs, const int64_t* track_offsets, int32_t n_predict,
                         int32_t em_iterations, double* pred_out, double* q_out, double* r_out, double* last_state_out,
                         std::vector<double>& buf) {
    const int64_t o0 = track_offsets[tr_i];
    const int T = (int)(track_offsets[tr_i + 1] - o0);
    if (T < 2) return "invalid argument: a track needs at least 2 observations (kalman.py:28-29)";
    if (buf.size() < (size_t)T * kFields) buf.resize((size_t)T * kFields);
    const TrackView t{buf.data(), 1};
    M4 Q;
    double R[2][2];
    V4 x;
    if (!kalman_fit(obs + 2 * o0, T, em_iterations, t, Q, R, x)) return "kalman: singular predicted covariance";
    rollout(x, n_predict, pred_out + (size_t)tr_i * n_predict * 2, nullptr, 0, Q, R);
    write_fit(tr_i, Q, R, x, q_out, r_out, last_state_out);
    return nullptr;
}

// One thread per track.  A singular predicted covariance (the host entry point's error) leaves NaN in every output of
// that track: the kernel never traps.
__global__ void __launch_bounds__(64) kalman_device_kernel(
        const double* __restrict__ obs, const int64_t* __restrict__ offs, int n_tracks, int n_predict,
        int em_iterations, int n_samples, const double* __restrict__ eps, double* __restrict__ pred,
        double* __restrict__ q_out, double* __restrict__ r_out, double* __restrict__ last_out, double* ws) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_tracks) return;
    const int64_t o0 = offs[i];
    const int T = (int)(offs[i + 1] - o0);
    const TrackView t{ws + i, n_tracks};
    M4 Q;
    double R[2][2];
    V4 x;
    double* p = pred + (int64_t)i * n_predict * 2;
    if (!kalman_fit(obs + 2 * o0, T, em_iterations, t, Q, R, x)) {
        const double nan = __longlong_as_double(0x7ff8000000000000LL);
        for (int k = 0; k < 2 * n_predict; ++k) p[k] = nan;
        for (int a = 0; a < 4; ++a) { x.a[a] = nan; for (int b = 0; b < 4; ++b) Q.a[a][b] = nan; }
        R[0][0] = R[0][1] = R[1][0] = R[1][1] = nan;
        write_fit(i, Q, R, x, q_out, r_out, last_out);
        return;
    }
    rollout(x, n_predict, p, (eps && n_samples > 0) ? eps + (int64_t)i * n_predict * 6 : nullptr, n_samples, Q, R);
    write_fit(i, Q, R, x, q_out, r_out, last_out);
}

constexpr int kKalmanThreads = 64;

int max_track_length(const int64_t* offs, int32_t n_tracks) {
    int64_t t_max = 0;
    for (int32_t i = 0; i < n_tracks; ++i) t_max = std::max(t_max, offs[i + 1] - offs[i]);
    return (int)t_max;
}

}  // namespace

extern "C" int tb2_kalman_predict(const double* obs, const int64_t* track_offsets, int32_t n_tracks,
                                  int32_t n_predict, int32_t em_iterations, double* pred_out,
                                  double* q_out, double* r_out, double* last_state_out) {
    TB2_REQUIRE(obs && track_offsets && pred_out && n_tracks >= 0 && n_predict >= 1 && em_iterations >= 0,
                "bad argument");
    // host threads over contiguous track ranges (TB2_KALMAN_THREADS overrides; small jobs stay on the calling thread)
    int threads = (int)std::thread::hardware_concurrency();
    if (const char* e = getenv("TB2_KALMAN_THREADS")) threads = atoi(e);
    threads = std::max(1, std::min(threads, n_tracks / 64));
    std::vector<const char*> errors((size_t)threads, nullptr);
    auto run = [&](int w) {
        std::vector<double> buf;
        const int lo = (int)((int64_t)n_tracks * w / threads), hi = (int)((int64_t)n_tracks * (w + 1) / threads);
        for (int i = lo; i < hi && !errors[w]; ++i)
            errors[w] = kalman_track(i, obs, track_offsets, n_predict, em_iterations, pred_out, q_out, r_out, last_state_out, buf);
    };
    if (threads == 1) run(0);
    else {
        std::vector<std::thread> pool;
        for (int w = 1; w < threads; ++w) pool.emplace_back(run, w);
        run(0);
        for (auto& th : pool) th.join();
    }
    for (const char* e : errors)
        if (e) { tb2::set_error(e); return TB2_ERR_INVALID; }
    return TB2_OK;
}

extern "C" size_t tb2_kalman_workspace_bytes(const int64_t* track_offsets_host, int32_t n_tracks) {
    if (!track_offsets_host || n_tracks <= 0) return 0;
    return (size_t)max_track_length(track_offsets_host, n_tracks) * kFields * (size_t)n_tracks * sizeof(double);
}

extern "C" int tb2_kalman_predict_device(const double* obs_dev, const int64_t* track_offsets_host,
                                         const int64_t* track_offsets_dev, int32_t n_tracks, int32_t n_predict,
                                         int32_t em_iterations, int32_t n_samples, const double* eps_dev,
                                         double* pred_out_dev, double* q_out_dev, double* r_out_dev,
                                         double* last_state_out_dev, void* workspace_dev, size_t workspace_bytes,
                                         void* stream) {
    TB2_REQUIRE(track_offsets_host && n_tracks >= 0 && n_predict >= 1 && em_iterations >= 0 && n_samples >= 0,
                "bad argument");
    TB2_REQUIRE(track_offsets_host[0] == 0, "track_offsets[0] must be 0");
    for (int32_t i = 0; i < n_tracks; ++i)
        TB2_REQUIRE(track_offsets_host[i + 1] - track_offsets_host[i] >= 2,
                    "a track needs at least 2 observations (kalman.py:28-29)");
    if (n_tracks == 0) return TB2_OK;
    TB2_REQUIRE(obs_dev && track_offsets_dev && pred_out_dev && workspace_dev, "null device pointer");
    TB2_REQUIRE(workspace_bytes >= tb2_kalman_workspace_bytes(track_offsets_host, n_tracks),
                "workspace smaller than tb2_kalman_workspace_bytes");
    cudaStream_t st = (cudaStream_t)stream;
    {
        tb2::KernelTimer kt("kalman_predict", st);
        kalman_device_kernel<<<(n_tracks + kKalmanThreads - 1) / kKalmanThreads, kKalmanThreads, 0, st>>>(
            obs_dev, track_offsets_dev, n_tracks, n_predict, em_iterations, n_samples, eps_dev, pred_out_dev, q_out_dev,
            r_out_dev, last_state_out_dev, (double*)workspace_dev);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}
