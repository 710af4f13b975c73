// Classical crowd simulators: social force and ORCA, one persistent rollout kernel and one sweep kernel for both.
//
// The reference builds ONE simulator per scene and crosses Python -> third-party code every
// step (classical/socialforce.py:89-95: 96 x socialforce.Simulator.step(); classical/orca.py:
// 99-119: 97 x rvo2 doStep() + 3 FFI calls per agent per step).  Here one CTA owns a scene for
// the whole rollout: the state lives in shared memory / registers for all steps, every
// pedestrian of the scene is a thread, the scenes of a batch run in lockstep in one launch,
// and only the sampled positions are written to HBM.
//
// Arithmetic follows the un-vendored upstream packages (socialforce v0.1.x: float64; RVO2
// v2.0.x: float) as restated in oracle/classical_oracle.py and oracle/orca_oracle.c -- parity
// vs upstream is UNPINNED (see those headers).  This file is compiled with -fmad=false so the
// CUDA result is comparable operation by operation with the CPU restatement.
#include <math_constants.h>

#include <cmath>
#include <type_traits>

#include "common.cuh"

namespace tb2 {

// =========================================================================================
// social force (double precision like upstream numpy)
// =========================================================================================
// The social-force code is written once over its scalar type T: double for the rollout itself, Dual for the rollout
// that also carries d/d(tau, v0, sigma) (tb2_sf_sweep_grad).

// Forward-mode dual number: a float64 value and its partials with respect to (tau, v0, sigma).  The value of every
// operation is the double operation on the values, so a Dual rollout's values equal the double rollout's bit for bit.
// Branches are taken by the caller on val(); their tangent is the taken branch's.
struct Dual {
    double v, d[3];
    Dual() = default;
    __device__ __forceinline__ Dual(double x) : v(x), d{0.0, 0.0, 0.0} {}

    __device__ __forceinline__ friend Dual operator+(const Dual& a, const Dual& b) {
        Dual r(a.v + b.v);
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = a.d[i] + b.d[i];
        return r;
    }
    __device__ __forceinline__ friend Dual operator+(const Dual& a, double b) {
        Dual r = a;
        r.v = a.v + b;
        return r;
    }
    __device__ __forceinline__ friend Dual operator-(const Dual& a, const Dual& b) {
        Dual r(a.v - b.v);
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = a.d[i] - b.d[i];
        return r;
    }
    __device__ __forceinline__ friend Dual operator-(double a, const Dual& b) {
        Dual r(a - b.v);
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = -b.d[i];
        return r;
    }
    __device__ __forceinline__ friend Dual operator-(const Dual& a) {
        Dual r(-a.v);
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = -a.d[i];
        return r;
    }
    __device__ __forceinline__ friend Dual operator*(const Dual& a, const Dual& b) {
        Dual r(a.v * b.v);
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = a.d[i] * b.v + a.v * b.d[i];
        return r;
    }
    __device__ __forceinline__ friend Dual operator*(double a, const Dual& b) {
        Dual r(a * b.v);
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = a * b.d[i];
        return r;
    }
    __device__ __forceinline__ friend Dual operator*(const Dual& a, double b) {
        Dual r(a.v * b);
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = a.d[i] * b;
        return r;
    }
    __device__ __forceinline__ friend Dual operator/(const Dual& a, const Dual& b) {
        Dual r(a.v / b.v);
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) / b.v;
        return r;
    }
    __device__ __forceinline__ friend Dual operator/(double a, const Dual& b) {
        Dual r(a / b.v);
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = -(r.v * b.d[i]) / b.v;
        return r;
    }
    __device__ __forceinline__ friend Dual operator/(const Dual& a, double b) {
        Dual r(a.v / b);
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = a.d[i] / b;
        return r;
    }
    __device__ __forceinline__ Dual& operator+=(const Dual& b) { return *this = *this + b; }
    // sqrt(0) occurs only as the norm of a zero vector, whose tangent is zero too: d = 0 there
    __device__ __forceinline__ friend Dual sqrt(const Dual& a) {
        Dual r(sqrt(a.v));
        const double k = r.v == 0.0 ? 0.0 : 0.5 / r.v;
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = a.d[i] * k;
        return r;
    }
    __device__ __forceinline__ friend Dual exp(const Dual& a) {
        Dual r(exp(a.v));
#pragma unroll
        for (int i = 0; i < 3; ++i) r.d[i] = r.v * a.d[i];
        return r;
    }
};
struct Dual2 { Dual x, y; };

__device__ __forceinline__ double val(double x) { return x; }
__device__ __forceinline__ double val(const Dual& x) { return x.v; }

// A swept parameter's unit tangent: parameter i of (tau, v0, sigma); nothing to seed in a double.
__device__ __forceinline__ void seed(double&, int) {}
__device__ __forceinline__ void seed(Dual& x, int i) { x.d[i] = 1.0; }

template <class T> struct Vec2Of { using type = double2; };
template <> struct Vec2Of<Dual> { using type = Dual2; };

template <class T>
struct SfScene {
    T* px; T* py; T* vx; T* vy; T* ex; T* ey; T* sp;
};

template <class T>
__device__ __forceinline__ T sf_potential(T rx, T ry, T sb, T ebx, T eby, double dt, T v0, T sigma) {
    // V(r_ab) = v0 exp(-b / sigma), b = 0.5 sqrt((|r| + |r - dt s_b e_b|)^2 - (dt s_b)^2)
    const T n1 = sqrt(rx * rx + ry * ry);
    const T qx = rx - dt * sb * ebx, qy = ry - dt * sb * eby;
    const T n2 = sqrt(qx * qx + qy * qy);
    const T s = n1 + n2;
    const T in_sqrt = s * s - (dt * sb) * (dt * sb);
    const T b = 0.5 * sqrt(in_sqrt);
    return v0 * exp(-b / sigma);
}

// One pedestrian of a social-force rollout: position, velocity, destination, initial and maximum speed
// (Simulator.__init__: initial_speeds, max_speeds = 1.3 x).  Destination and speeds do not depend on the parameters.
template <class T>
struct SfAgent { T x, y, ux, uy; double dx, dy, s0, smax; };

template <class T>
__device__ __forceinline__ SfAgent<T> sf_agent_init(const double* st) {
    SfAgent<T> g;
    g.x = st[0]; g.y = st[1]; g.ux = st[2]; g.uy = st[3]; g.dx = st[4]; g.dy = st[5];
    g.s0 = sqrt(val(g.ux) * val(g.ux) + val(g.uy) * val(g.uy));
    g.smax = 1.3 * g.s0;
    return g;
}

__device__ __forceinline__ double sf_cosphi() { return cos(200.0 / 2.0 / 180.0 * 3.141592653589793); }   // FieldOfView(twophi=200)

// First half of a step: the desired direction (NaN at the destination, as upstream), published with the state for the
// neighbour loop of every pedestrian of the scene.
template <class T>
__device__ __forceinline__ void sf_publish(const SfAgent<T>& g, const SfScene<T>& sc, int a, T& eax, T& eay) {
    const T gx = g.dx - g.x, gy = g.dy - g.y;
    const T gn = sqrt(gx * gx + gy * gy);
    eax = gx / gn; eay = gy / gn;
    sc.px[a] = g.x; sc.py[a] = g.y; sc.vx[a] = g.ux; sc.vy[a] = g.uy; sc.ex[a] = eax; sc.ey[a] = eay;
    sc.sp[a] = sqrt(g.ux * g.ux + g.uy * g.uy);
}

// Second half: driving force + pairwise repulsion over b = 0 .. n-1 in index order, speed clip, position update.
// The field-of-view test and the clip take their branch from the value.
template <class T>
__device__ __forceinline__ void sf_advance(SfAgent<T>& g, const SfScene<T>& sc, int a, int n, T eax, T eay, double dt,
                                           T tau, T v0, T sigma, double cosphi) {
    const double fd = 1e-3;
    T Fx = 1.0 / tau * (g.s0 * eax - g.ux);
    T Fy = 1.0 / tau * (g.s0 * eay - g.uy);
    T sumx = 0.0, sumy = 0.0;
    for (int b = 0; b < n; ++b) {
        T fx = 0.0, fy = 0.0;
        double w = 0.0;
        if (b != a) {
            const T rx = g.x - sc.px[b], ry = g.y - sc.py[b];
            const T sb = sc.sp[b], ebx = sc.ex[b], eby = sc.ey[b];
            const T v = sf_potential(rx, ry, sb, ebx, eby, dt, v0, sigma);
            const T dvdx = (sf_potential(rx + fd, ry, sb, ebx, eby, dt, v0, sigma) - v) / fd;
            const T dvdy = (sf_potential(rx, ry + fd, sb, ebx, eby, dt, v0, sigma) - v) / fd;
            fx = -1.0 * dvdx; fy = -1.0 * dvdy;               // f_ab = -grad V
            const T gx = -fx, gy = -fy;                       // w(e, -f_ab)
            const bool in_sight = val(eax * gx + eay * gy) > val(sqrt(gx * gx + gy * gy) * cosphi);
            w = in_sight ? 1.0 : 0.5;
        }
        sumx += w * fx;
        sumy += w * fy;
    }
    Fx += sumx; Fy += sumy;
    const T wx = g.ux + dt * Fx, wy = g.uy + dt * Fy;
    const T wn = sqrt(wx * wx + wy * wy);
    const T q = g.smax / wn;
    const T factor = isnan(val(q)) ? q : (val(q) < 1.0 ? q : T(1.0));      // numpy.minimum(1, q)
    g.ux = wx * factor; g.uy = wy * factor;
    g.x = g.x + g.ux * dt; g.y = g.y + g.uy * dt;
}

// =========================================================================================
// ORCA (float like RVO2)
// =========================================================================================
constexpr int kOrcaMaxNeigh = 16;
constexpr float kOrcaEps = 0.00001f;

struct Line { float2 point, dir; };

__device__ __forceinline__ float2 f2(float x, float y) { return make_float2(x, y); }
__device__ __forceinline__ float2 vadd(float2 a, float2 b) { return f2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 vsub(float2 a, float2 b) { return f2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 vmul(float s, float2 a) { return f2(s * a.x, s * a.y); }
__device__ __forceinline__ float vdot(float2 a, float2 b) { return a.x * b.x + a.y * b.y; }
__device__ __forceinline__ float vdet(float2 a, float2 b) { return a.x * b.y - a.y * b.x; }
__device__ __forceinline__ float vabssq(float2 a) { return vdot(a, a); }
__device__ __forceinline__ float2 vnormalize(float2 a) {
    float l = sqrtf(vabssq(a));
    return f2(a.x / l, a.y / l);
}

__device__ bool orca_lp1(const Line* lines, int line_no, float radius, float2 opt, bool dir_opt, float2& result) {
    const float dp = vdot(lines[line_no].point, lines[line_no].dir);
    const float disc = dp * dp + radius * radius - vabssq(lines[line_no].point);
    if (disc < 0.0f) return false;
    const float sq = sqrtf(disc);
    float t_left = -dp - sq, t_right = -dp + sq;
    for (int i = 0; i < line_no; ++i) {
        const float den = vdet(lines[line_no].dir, lines[i].dir);
        const float num = vdet(lines[i].dir, vsub(lines[line_no].point, lines[i].point));
        if (fabsf(den) <= kOrcaEps) {
            if (num < 0.0f) return false;
            continue;
        }
        const float t = num / den;
        if (den >= 0.0f) t_right = fminf(t_right, t); else t_left = fmaxf(t_left, t);
        if (t_left > t_right) return false;
    }
    if (dir_opt) {
        if (vdot(opt, lines[line_no].dir) > 0.0f) result = vadd(lines[line_no].point, vmul(t_right, lines[line_no].dir));
        else result = vadd(lines[line_no].point, vmul(t_left, lines[line_no].dir));
    } else {
        const float t = vdot(lines[line_no].dir, vsub(opt, lines[line_no].point));
        if (t < t_left) result = vadd(lines[line_no].point, vmul(t_left, lines[line_no].dir));
        else if (t > t_right) result = vadd(lines[line_no].point, vmul(t_right, lines[line_no].dir));
        else result = vadd(lines[line_no].point, vmul(t, lines[line_no].dir));
    }
    return true;
}

__device__ int orca_lp2(const Line* lines, int n, float radius, float2 opt, bool dir_opt, float2& result) {
    if (dir_opt) result = vmul(radius, opt);
    else if (vabssq(opt) > radius * radius) result = vmul(radius, vnormalize(opt));
    else result = opt;
    for (int i = 0; i < n; ++i) {
        if (vdet(lines[i].dir, vsub(lines[i].point, result)) > 0.0f) {
            const float2 tmp = result;
            if (!orca_lp1(lines, i, radius, opt, dir_opt, result)) {
                result = tmp;
                return i;
            }
        }
    }
    return n;
}

__device__ void orca_lp3(const Line* lines, int n, int begin, float radius, float2& result) {
    float distance = 0.0f;
    Line proj[kOrcaMaxNeigh];
    for (int i = begin; i < n; ++i) {
        if (vdet(lines[i].dir, vsub(lines[i].point, result)) > distance) {
            int np = 0;
            for (int j = 0; j < i; ++j) {
                Line l;
                const float d = vdet(lines[i].dir, lines[j].dir);
                if (fabsf(d) <= kOrcaEps) {
                    if (vdot(lines[i].dir, lines[j].dir) > 0.0f) continue;
                    l.point = vmul(0.5f, vadd(lines[i].point, lines[j].point));
                } else {
                    l.point = vadd(lines[i].point,
                                   vmul(vdet(lines[j].dir, vsub(lines[i].point, lines[j].point)) / d, lines[i].dir));
                }
                l.dir = vnormalize(vsub(lines[j].dir, lines[i].dir));
                proj[np++] = l;
            }
            const float2 tmp = result;
            if (orca_lp2(proj, np, radius, f2(-lines[i].dir.y, lines[i].dir.x), true, result) < np) result = tmp;
            distance = vdet(lines[i].dir, vsub(lines[i].point, result));
        }
    }
}

// One ORCA agent: position and velocity (float, like RVO2), preferred velocity, goal and initial speed (double, like the
// reference's numpy code), maximum speed 1.3 x the initial speed (orca.py:36,55  MAX_SPEED_MULTIPLIER).
struct OrcaAgent { float2 pos, vel, pref; double2 goal; double speed; float maxsp; };

__device__ __forceinline__ OrcaAgent orca_agent_init(float2 pos, float2 vel, double2 goal, double speed) {
    OrcaAgent g;
    g.pos = pos; g.vel = vel; g.pref = f2(0.f, 0.f); g.goal = goal; g.speed = speed;
    g.maxsp = (float)(1.3 * speed);
    return g;
}

// Per-setting constants of a step (RVO2 computeNewVelocity).
struct OrcaStep {
    float range_sq, inv_th, inv_ts, cr, crsq;
    int max_nb;
};

__device__ __forceinline__ OrcaStep orca_step_consts(float time_step, float neighbor_dist, float time_horizon, float radius,
                                                     int max_nb) {
    OrcaStep c;
    c.inv_th = 1.0f / time_horizon;
    c.inv_ts = 1.0f / time_step;
    c.cr = radius + radius;
    c.crsq = c.cr * c.cr;
    c.range_sq = neighbor_dist * neighbor_dist;
    c.max_nb = max_nb;
    return c;
}

// First half of a step: the new velocity of agent a from the scene's published positions / velocities (neighbours
// b = 0 .. n-1 in index order, ORCA lines, linear programs 2 and 3).
__device__ __forceinline__ float2 orca_new_velocity(const float2* pos, const float2* vel, int a, int n, const OrcaAgent& g,
                                                    const OrcaStep& c) {
    const float2 mypos = g.pos, myvel = g.vel;
    int nb[kOrcaMaxNeigh];
    float nd[kOrcaMaxNeigh];
    int nn = 0;
    float range_sq = c.range_sq;
    for (int b = 0; b < n; ++b) {
        if (b == a) continue;
        const float dsq = vabssq(vsub(mypos, pos[b]));
        if (dsq < range_sq) {
            if (nn < c.max_nb) { nb[nn] = b; nd[nn] = dsq; ++nn; }
            int i = nn - 1;
            while (i != 0 && dsq < nd[i - 1]) { nb[i] = nb[i - 1]; nd[i] = nd[i - 1]; --i; }
            nb[i] = b; nd[i] = dsq;
            if (nn == c.max_nb) range_sq = nd[nn - 1];
        }
    }
    Line lines[kOrcaMaxNeigh];
    for (int k = 0; k < nn; ++k) {
        const int b = nb[k];
        const float2 rp = vsub(pos[b], mypos);
        const float2 rv = vsub(myvel, vel[b]);
        const float dsq = vabssq(rp);
        Line l;
        float2 u;
        if (dsq > c.crsq) {
            const float2 w = vsub(rv, vmul(c.inv_th, rp));
            const float wsq = vabssq(w);
            const float dp1 = vdot(w, rp);
            if (dp1 < 0.0f && dp1 * dp1 > c.crsq * wsq) {
                const float wl = sqrtf(wsq);
                const float2 uw = f2(w.x / wl, w.y / wl);
                l.dir = f2(uw.y, -uw.x);
                u = vmul(c.cr * c.inv_th - wl, uw);
            } else {
                const float leg = sqrtf(dsq - c.crsq);
                if (vdet(rp, w) > 0.0f) {
                    l.dir = f2((rp.x * leg - rp.y * c.cr) / dsq, (rp.x * c.cr + rp.y * leg) / dsq);
                } else {
                    l.dir = f2(-(rp.x * leg + rp.y * c.cr) / dsq, -(-rp.x * c.cr + rp.y * leg) / dsq);
                }
                const float dp2 = vdot(rv, l.dir);
                u = vsub(vmul(dp2, l.dir), rv);
            }
        } else {
            const float2 w = vsub(rv, vmul(c.inv_ts, rp));
            const float wl = sqrtf(vabssq(w));
            const float2 uw = f2(w.x / wl, w.y / wl);
            l.dir = f2(uw.y, -uw.x);
            u = vmul(c.cr * c.inv_ts - wl, uw);
        }
        l.point = vadd(myvel, vmul(0.5f, u));
        lines[k] = l;
    }
    float2 res;
    const int fail = orca_lp2(lines, nn, g.maxsp, g.pref, false, res);
    if (fail < nn) orca_lp3(lines, nn, fail, g.maxsp, res);
    return res;
}

// Second half: take the new velocity, move, and steer the preferred velocity at the goal (orca.py:111-119, double like
// the reference's numpy code).
__device__ __forceinline__ void orca_advance(OrcaAgent& g, float2 newv, float time_step, double end_range) {
    g.vel = newv;
    g.pos = vadd(g.pos, vmul(time_step, g.vel));
    const double gx = g.goal.x - (double)g.pos.x, gy = g.goal.y - (double)g.pos.y;
    const double dist = sqrt(gx * gx + gy * gy);
    if (dist < end_range) g.pref = f2(0.f, 0.f);
    else if (dist > g.speed) g.pref = f2((float)(g.speed * gx / dist), (float)(g.speed * gy / dist));
    else g.pref = f2((float)gx, (float)gy);
}

// =========================================================================================
// One rollout for both simulators
// =========================================================================================
// A simulator trait holds what differs between social force and ORCA: the agent and its initial state, the constants
// of a setting (the params struct, or a sweep's [3] settings row in place of its three swept fields), the scene arrays
// in shared memory, a prologue before the first step, the two phases of a step around the scene barrier (phase 1 reads
// the scene, phase 2 moves the agent), which step counts take a sample, and the host-side checks of its parameters.

// kWarpScenes: every scene has at most 32 pedestrians -> one WARP per scene, 4 scenes per CTA, __syncwarp instead
// of __syncthreads (a CTA of one warp caps an SM at 32 resident warps; the arithmetic per pedestrian is unchanged,
// results are bit-identical to the one-scene-per-CTA form).
constexpr int kScenesPerCta = 4;

template <bool kWarpScenes>
__device__ __forceinline__ void scene_sync() {
    if (kWarpScenes) __syncwarp();
    else __syncthreads();
}

// Social force over scalar type T; SfSim (double) is the rollout, SfGradSim (Dual) the rollout with its tangents.
template <class T>
struct SfRollout {
    using Params = tb2_sf_params;
    using Setting = double;                    // tau, v0, sigma
    using Agent = SfAgent<T>;
    using Scene = SfScene<T>;
    using Handoff = typename Vec2Of<T>::type;  // phase 1 -> phase 2: the desired direction
    using Pos = typename Vec2Of<T>::type;
    struct Inputs { const double* state; };
    struct Consts { double dt; T tau, v0, sigma; double cosphi; };
    static constexpr size_t kPedBytes = 7 * sizeof(T);
    static constexpr int kSampleOffset = 0;    // sample after step k = 0 .. n_steps - 1 when k % sample_every == 0

    __device__ static Agent agent(const Inputs& in, int row) { return sf_agent_init<T>(in.state + (size_t)row * 6); }
    // The swept parameters seeded with unit tangents (for T = Dual).
    __device__ static Consts consts(const Params& p, const Setting* row) {
        Consts c = {(double)p.delta_t, row ? row[0] : (double)p.tau, row ? row[1] : (double)p.v0,
                    row ? row[2] : (double)p.sigma, sf_cosphi()};
        seed(c.tau, 0); seed(c.v0, 1); seed(c.sigma, 2);
        return c;
    }
    // The scene arrays from pedestrian slot `first` on, each `stride` long.
    __device__ static Scene scene(void* arrays, size_t first, int stride) {
        T* px = static_cast<T*>(arrays) + first * 7;
        return {px, px + stride, px + 2 * stride, px + 3 * stride, px + 4 * stride, px + 5 * stride, px + 6 * stride};
    }
    template <bool kWarp>
    __device__ static void prologue(const Agent&, const Scene&, int, bool) {}
    __device__ static Handoff phase1(const Agent& g, const Consts&, const Scene& sc, int a, int) {
        Handoff e;
        sf_publish(g, sc, a, e.x, e.y);
        return e;
    }
    __device__ static void phase2(Agent& g, const Consts& c, const Scene& sc, int a, int n, Handoff e) {
        sf_advance(g, sc, a, n, e.x, e.y, c.dt, c.tau, c.v0, c.sigma, c.cosphi);
    }
    __device__ static Pos position(const Agent& g) { return {g.x, g.y}; }

    static int check(const Params&) { return TB2_OK; }
    static int check_setting(const Setting* s) {
        TB2_REQUIRE(s[0] > 0.0 && s[2] > 0.0, "tau and sigma must be > 0");
        return TB2_OK;
    }
};

struct SfSim : SfRollout<double> {};
struct SfGradSim : SfRollout<Dual> {};

struct OrcaSim {
    using Params = tb2_orca_params;
    using Setting = float;                     // neighbor_dist, time_horizon, radius
    using Agent = OrcaAgent;
    struct Scene { float2* pos; float2* vel; };
    using Handoff = float2;                    // phase 1 -> phase 2: the new velocity
    using Pos = float2;
    struct Inputs { const float2* pos; const float2* vel; const double2* goal; const double* speed; };
    struct Consts { OrcaStep step; float time_step; double end_range; };
    static constexpr size_t kPedBytes = 2 * sizeof(float2);
    static constexpr int kSampleOffset = 1;    // sample after step count = 1 .. n_steps when count % sample_every == 0

    __device__ static Agent agent(const Inputs& in, int row) {
        return orca_agent_init(in.pos[row], in.vel[row], in.goal[row], in.speed[row]);
    }
    __device__ static Consts consts(const Params& p, const Setting* row) {
        return {orca_step_consts(p.time_step, row ? row[0] : p.neighbor_dist, row ? row[1] : p.time_horizon,
                                 row ? row[2] : p.radius, p.max_neighbors),
                p.time_step, p.end_range};
    }
    __device__ static Scene scene(void* arrays, size_t first, int stride) {
        float2* pos = static_cast<float2*>(arrays) + first * 2;
        return {pos, pos + stride};
    }
    // The first step reads every agent's initial position / velocity.
    template <bool kWarp>
    __device__ static void prologue(const Agent& g, const Scene& sc, int a, bool on) {
        if (on) { sc.pos[a] = g.pos; sc.vel[a] = g.vel; }
        scene_sync<kWarp>();
    }
    __device__ static Handoff phase1(const Agent& g, const Consts& c, const Scene& sc, int a, int n) {
        return orca_new_velocity(sc.pos, sc.vel, a, n, g, c.step);
    }
    __device__ static void phase2(Agent& g, const Consts& c, const Scene& sc, int a, int, Handoff v) {
        orca_advance(g, v, c.time_step, c.end_range);
        sc.pos[a] = g.pos;
        sc.vel[a] = g.vel;
    }
    __device__ static Pos position(const Agent& g) { return g.pos; }

    static int check(const Params& p) {
        TB2_REQUIRE(p.max_neighbors >= 1 && p.max_neighbors <= kOrcaMaxNeigh, "max_neighbors must be in [1, 16]");
        return TB2_OK;
    }
    static int check_setting(const Setting* s) {
        TB2_REQUIRE(s[1] > 0.0f && s[2] > 0.0f, "time_horizon and radius must be > 0");
        return TB2_OK;
    }
};

// Samples of an n_steps rollout: the step counts k = kSampleOffset .. n_steps - 1 + kSampleOffset that `every` divides.
template <class Sim>
__host__ __device__ __forceinline__ int sample_count(int n_steps, int every) {
    return (n_steps - 1 + Sim::kSampleOffset) / every + 1 - Sim::kSampleOffset;
}

// The rollout of agent a of a scene of n under one setting.  Lanes with on == false (no pedestrian, or no setting)
// take only the barriers.  sink(sample, position) receives, in sample order, the samples of the lanes it takes.
template <class Sim, bool kWarp, class Sink>
__device__ __forceinline__ void rollout(typename Sim::Agent g, const typename Sim::Consts& c,
                                        const typename Sim::Scene& sc, int a, int n, bool on, int n_steps, int every,
                                        Sink& sink) {
    Sim::template prologue<kWarp>(g, sc, a, on);
    int sample = 0;
    for (int k = Sim::kSampleOffset; k < n_steps + Sim::kSampleOffset; ++k) {
        typename Sim::Handoff h = {};
        if (on) h = Sim::phase1(g, c, sc, a, n);
        scene_sync<kWarp>();                       // every agent has read the scene before any agent moves
        if (on) Sim::phase2(g, c, sc, a, n, h);
        if (k % every == 0) {
            if (on && sink.takes(a)) sink(sample, Sim::position(g));
            ++sample;
        }
        scene_sync<kWarp>();
    }
}

// Sample j of every pedestrian -> out[j * A + row].
template <class Pos>
struct PositionSink {
    __device__ static bool takes(int) { return true; }
    Pos* out;
    int A, row;
    __device__ void operator()(int sample, Pos pos) const { out[(size_t)sample * A + row] = pos; }
};

// The primary's (pedestrian 0's) score against the truth rows tr: |truth - position| in float64 (ORCA's float position
// widened first, the adapter's astype(np.float64)), summed in sample order; `last` is the final distance.
struct ScoreSink {
    __device__ static bool takes(int a) { return a == 0; }
    const double* tr;
    double sum = 0.0, last = 0.0;
    template <class Pos>
    __device__ void operator()(int sample, Pos pos) {
        const double ex = tr[2 * sample] - (double)pos.x, ey = tr[2 * sample + 1] - (double)pos.y;
        last = sqrt(ex * ex + ey * ey);
        sum += last;
    }
};

// ScoreSink for a Dual rollout: the same values, and d|truth - position| with them, in sample order.
struct GradScoreSink {
    __device__ static bool takes(int a) { return a == 0; }
    const double* tr;
    Dual sum = 0.0, last = 0.0;
    __device__ void operator()(int sample, const Dual2& pos) {
        const Dual ex = tr[2 * sample] - pos.x, ey = tr[2 * sample + 1] - pos.y;
        last = sqrt(ex * ex + ey * ey);
        sum += last;
    }
};

// Launch bounds: the CTA form takes scenes of up to 1024 pedestrians, one thread each, so it must compile to at most 64
// registers a thread (65 536 / 1024); unbounded, ptxas gave social force 80 and the device refused blocks above 768
// threads.  The warp form keeps its fixed 128-thread CTA.  minBlocks = 1 leaves the warp form's register budget where
// it was (with 128 alone it spilled).
template <class Sim, bool kWarpScenes>
__global__ void __launch_bounds__(kWarpScenes ? 32 * kScenesPerCta : 1024, 1)
simulate_kernel(const int* __restrict__ scene_off, typename Sim::Inputs in, typename Sim::Pos* __restrict__ out, int A,
                int B, int n_max, typename Sim::Params p) {
    extern __shared__ double smem_classical[];
    const int scene = kWarpScenes ? blockIdx.x * kScenesPerCta + (int)(threadIdx.x >> 5) : (int)blockIdx.x;
    if (scene >= B) return;                                  // whole warp (kWarpScenes): no block-wide barrier below
    const int row0 = scene_off[scene];
    const int n = scene_off[scene + 1] - row0;
    const int a = kWarpScenes ? (int)(threadIdx.x & 31) : (int)threadIdx.x;
    const typename Sim::Scene sc = Sim::scene(smem_classical, kWarpScenes ? (size_t)(threadIdx.x >> 5) * n_max : 0, n);
    typename Sim::Agent g = {};
    if (a < n) g = Sim::agent(in, row0 + a);
    PositionSink<typename Sim::Pos> sink{out, A, row0 + a};
    rollout<Sim, kWarpScenes>(g, Sim::consts(p, nullptr), sc, a, n, a < n, p.n_steps, p.sample_every, sink);
}

// -----------------------------------------------------------------------------------------
// Parameter sweeps: a work item is (scene, setting); only the primary's ADE / FDE leave the chip.
// One CTA per scene runs every setting of it.  kPacked (scene of n <= 32): lane segments of W = next power of two >= n,
// each segment its own setting with its own scene arrays, 32 / W settings per warp in lockstep under __syncwarp.
// Otherwise the whole CTA is one item, looping over the settings.  Each thread keeps its pedestrian's initial state in
// registers (the lane -> pedestrian map is fixed for the scene); the primary's truth sits in shared memory.  The primary
// (pedestrian 0) accumulates |truth - position| in float64, sequentially over the samples: ADE = sum / n_samples,
// FDE = the last distance.  No atomics: reruns are bit-identical.
// -----------------------------------------------------------------------------------------
constexpr int kSweepWarps = 4;

__device__ __forceinline__ int sweep_width(int n) {
    int w = 1;
    while (w < n) w <<= 1;
    return w;
}

// Lane geometry of one item: pedestrian index a, first setting `slot`, settings per round `nslots`, array stride.
struct SweepLane { int a, slot, nslots, stride, warp_first; };

template <bool kPacked>
__device__ __forceinline__ SweepLane sweep_lane(int n) {
    SweepLane L;
    if (kPacked) {
        const int W = sweep_width(n), per_warp = 32 / W, lane = (int)(threadIdx.x & 31), warp = (int)(threadIdx.x >> 5);
        L.a = lane & (W - 1);
        L.warp_first = warp * per_warp;
        L.slot = L.warp_first + lane / W;
        L.nslots = (int)(blockDim.x >> 5) * per_warp;
        L.stride = W;
    } else {
        L.a = (int)threadIdx.x;
        L.warp_first = L.slot = 0;
        L.nslots = 1;
        L.stride = n;
    }
    return L;
}

// Loads the primary's last n_samples truth rows into shared memory; returns false when the CTA's scene is not of
// this form (packed: n <= 32; CTA: n > 32).
template <bool kPacked>
__device__ __forceinline__ bool sweep_scene(const int* scene_off, const double* truth, int T, int n_samples,
                                            double* tr, int& row0, int& n) {
    row0 = scene_off[blockIdx.x];
    n = scene_off[blockIdx.x + 1] - row0;
    if (kPacked ? n > 32 : n <= 32) return false;            // whole CTA
    const double* src = truth + ((size_t)blockIdx.x * T + (T - n_samples)) * 2;
    for (int i = (int)threadIdx.x; i < 2 * n_samples; i += (int)blockDim.x) tr[i] = src[i];
    __syncthreads();
    return true;
}

// params [P, 3]: row s replaces the three swept fields of p (SfSim / OrcaSim::Setting).  Launch bounds as for
// simulate_kernel: the CTA form up to 1024 threads, the packed form at most kSweepWarps warps.
template <class Sim, bool kPacked>
__global__ void __launch_bounds__(kPacked ? 32 * kSweepWarps : 1024, 1)
sweep_kernel(const int* __restrict__ scene_off, typename Sim::Inputs in, const typename Sim::Setting* __restrict__ params,
             int P, const double* __restrict__ truth, int T, double* __restrict__ ade, double* __restrict__ fde, int B,
             typename Sim::Params p) {
    extern __shared__ double smem_classical[];
    const int n_samples = sample_count<Sim>(p.n_steps, p.sample_every);
    double* tr = smem_classical;
    int row0, n;
    if (!sweep_scene<kPacked>(scene_off, truth, T, n_samples, tr, row0, n)) return;
    const SweepLane L = sweep_lane<kPacked>(n);
    // this segment's arrays: packed, the segment's first lane is its first pedestrian
    const typename Sim::Scene sc = Sim::scene(tr + 2 * n_samples, kPacked ? threadIdx.x - L.a : 0, L.stride);
    typename Sim::Agent g0 = {};
    if (L.a < n) g0 = Sim::agent(in, row0 + L.a);
    for (int base = 0; base < P; base += L.nslots) {
        if (kPacked && base + L.warp_first >= P) break;     // warp-uniform: no setting left for this warp
        const int s = base + L.slot;
        const bool on = L.a < n && s < P;
        ScoreSink sink{tr};
        rollout<Sim, kPacked>(g0, Sim::consts(p, on ? params + (size_t)s * 3 : nullptr), sc, L.a, n, on, p.n_steps,
                              p.sample_every, sink);
        if (on && L.a == 0) {
            ade[(size_t)s * B + blockIdx.x] = sink.sum / (double)n_samples;
            fde[(size_t)s * B + blockIdx.x] = sink.last;
        }
    }
}

// The tangent sweep: sweep_kernel<SfGradSim> with GradScoreSink, writing dade / dfde [P, B, 3] (d/d(tau, v0, sigma) of
// each item's ADE / FDE) beside ade / fde.  Its own kernel rather than an output policy of sweep_kernel, which would
// change the value kernels' register schedule.  A Dual rollout needs about four times the registers of the double one:
// the CTA form is bounded at kSfGradMaxScene threads, which ptxas fits in 255 registers without spills.
constexpr int kSfGradMaxScene = 256;

template <bool kPacked>
__global__ void __launch_bounds__(kPacked ? 32 * kSweepWarps : kSfGradMaxScene, 1)
sf_sweep_grad_kernel(const int* __restrict__ scene_off, SfGradSim::Inputs in, const double* __restrict__ params, int P,
                     const double* __restrict__ truth, int T, double* __restrict__ ade, double* __restrict__ fde,
                     double* __restrict__ dade, double* __restrict__ dfde, int B, SfGradSim::Params p) {
    extern __shared__ double smem_classical[];
    const int n_samples = sample_count<SfGradSim>(p.n_steps, p.sample_every);
    double* tr = smem_classical;
    int row0, n;
    if (!sweep_scene<kPacked>(scene_off, truth, T, n_samples, tr, row0, n)) return;
    const SweepLane L = sweep_lane<kPacked>(n);
    const SfGradSim::Scene sc = SfGradSim::scene(tr + 2 * n_samples, kPacked ? threadIdx.x - L.a : 0, L.stride);
    SfGradSim::Agent g0 = {};
    if (L.a < n) g0 = SfGradSim::agent(in, row0 + L.a);
    for (int base = 0; base < P; base += L.nslots) {
        if (kPacked && base + L.warp_first >= P) break;
        const int s = base + L.slot;
        const bool on = L.a < n && s < P;
        GradScoreSink sink{tr};
        rollout<SfGradSim, kPacked>(g0, SfGradSim::consts(p, on ? params + (size_t)s * 3 : nullptr), sc, L.a, n, on,
                                    p.n_steps, p.sample_every, sink);
        if (on && L.a == 0) {
            const size_t i = (size_t)s * B + blockIdx.x;
            const Dual m = sink.sum / (double)n_samples;
            ade[i] = m.v;
            fde[i] = sink.last.v;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                dade[i * 3 + j] = m.d[j];
                dfde[i * 3 + j] = sink.last.d[j];
            }
        }
    }
}

}  // namespace tb2

using namespace tb2;

template <class Sim>
static int check_rollout(const typename Sim::Params& p) {
    TB2_REQUIRE(p.n_steps >= 1 && p.sample_every >= 1, "bad step counts");
    return Sim::check(p);
}

// Warp form (4 scenes per 128-thread CTA) when every scene has at most 32 pedestrians, else one CTA per scene.
template <class Sim>
static int simulate_launch(const char* name, const tb2_layout* l, const typename Sim::Params& p,
                           typename Sim::Inputs in, typename Sim::Pos* out, void* stream) {
    int rc = check_rollout<Sim>(p);
    if (rc != TB2_OK) return rc;
    TB2_REQUIRE(l->n_max <= 1024, "scene larger than 1024 pedestrians");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = (size_t)l->n_max * Sim::kPedBytes;
    {
        KernelTimer kt(name, st);
        if (l->n_max <= 32)
            simulate_kernel<Sim, true><<<(l->B + kScenesPerCta - 1) / kScenesPerCta, 32 * kScenesPerCta,
                                         smem * kScenesPerCta, st>>>(l->scene_off, in, out, l->M, l->B, l->n_max, p);
        else {
            static DynSmemConfig configured;
            TB2_CHECK_CUDA(configured.ensure(simulate_kernel<Sim, false>, smem, 48 * 1024));
            simulate_kernel<Sim, false><<<l->B, (l->n_max + 31) / 32 * 32, smem, st>>>(l->scene_off, in, out, l->M,
                                                                                      l->B, l->n_max, p);
        }
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// Host-side checks shared by the sweeps: counts, then the parameters read back from the device (P x 3 values).
template <typename T>
static int sweep_params_host(const T* params_dev, int P, std::vector<T>& h, cudaStream_t st) {
    h.resize((size_t)P * 3);
    TB2_CHECK_CUDA(cudaMemcpyAsync(h.data(), params_dev, h.size() * sizeof(T), cudaMemcpyDeviceToHost, st));
    TB2_CHECK_CUDA(cudaStreamSynchronize(st));
    for (T v : h) TB2_REQUIRE(isfinite((double)v), "non-finite sweep parameter");
    return TB2_OK;
}

static int sweep_counts(const tb2_layout* l, int P, int T, int n_samples, int max_scene) {
    TB2_REQUIRE(l->B >= 1, "no scenes");
    TB2_REQUIRE(P >= 1, "P < 1 settings");
    TB2_REQUIRE((int64_t)P * l->B < ((int64_t)1 << 31), "P x B >= 2^31");
    TB2_REQUIRE(l->n_max <= max_scene, "scene larger than " + std::to_string(max_scene) + " pedestrians");
    TB2_REQUIRE(n_samples >= 1 && n_samples <= 1024, "sample count must be in [1, 1024]");
    TB2_REQUIRE(T >= n_samples, "truth shorter than the sample count");
    return TB2_OK;
}

// Checks the call, then launches both forms over every scene; each CTA keeps only the scenes of its form (packed:
// n <= 32, CTA: n > 32).  launch(form, threads, smem) launches the kernel of form std::true_type (packed) or
// std::false_type (CTA) on B CTAs.
template <class Sim, class Launch>
static int sweep_launch(const char* name, const tb2_layout* l, const typename Sim::Params& p,
                        const typename Sim::Setting* params, int P, int T, int max_scene, void* stream, Launch launch) {
    int rc = check_rollout<Sim>(p);
    if (rc != TB2_OK) return rc;
    const int n_samples = sample_count<Sim>(p.n_steps, p.sample_every);
    rc = sweep_counts(l, P, T, n_samples, max_scene);
    if (rc != TB2_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<typename Sim::Setting> h;
    rc = sweep_params_host(params, P, h, st);
    for (int s = 0; rc == TB2_OK && s < P; ++s) rc = Sim::check_setting(&h[(size_t)s * 3]);
    if (rc != TB2_OK) return rc;

    const size_t truth_bytes = (size_t)n_samples * 2 * sizeof(double);
    const int w_max = l->n_max >= 32 ? 32 : (l->n_max <= 1 ? 1 : 1 << (32 - __builtin_clz(l->n_max - 1)));
    const int64_t want = ((int64_t)P * w_max + 31) / 32;
    const int warps = (int)(want < kSweepWarps ? want : kSweepWarps);
    KernelTimer kt(name, st);
    rc = launch(std::true_type(), 32 * warps, truth_bytes + (size_t)32 * warps * Sim::kPedBytes, st);
    if (rc != TB2_OK) return rc;
    if (l->n_max > 32)
        rc = launch(std::false_type(), (l->n_max + 31) / 32 * 32, truth_bytes + (size_t)l->n_max * Sim::kPedBytes, st);
    return rc;
}

// One sweep kernel form: dynamic shared memory above 48 KB opted into once per kernel and device.
template <class Kernel, class... Args>
static int sweep_form(Kernel kernel, DynSmemConfig& configured, int B, int threads, size_t smem, cudaStream_t st,
                      Args... args) {
    TB2_CHECK_CUDA(configured.ensure(kernel, smem, 48 * 1024));
    kernel<<<B, threads, smem, st>>>(args...);
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

template <class Sim>
static int sweep_values(const char* name, const tb2_layout* l, const typename Sim::Params& p,
                        const typename Sim::Setting* params, int P, typename Sim::Inputs in, const double* truth, int T,
                        double* ade, double* fde, void* stream) {
    return sweep_launch<Sim>(name, l, p, params, P, T, 1024, stream, [&](auto packed, int threads, size_t smem,
                                                                            cudaStream_t st) {
        static DynSmemConfig configured;
        return sweep_form(sweep_kernel<Sim, decltype(packed)::value>, configured, l->B, threads, smem, st, l->scene_off,
                          in, params, P, truth, T, ade, fde, l->B, p);
    });
}

extern "C" {

int tb2_sf_simulate(const tb2_layout* l, const tb2_sf_params* p, const double* state, double* out, void* stream) {
    TB2_REQUIRE(l && p && state && out, "null argument");
    return simulate_launch<SfSim>("sf_simulate", l, *p, {state}, (double2*)out, stream);
}

int tb2_orca_simulate(const tb2_layout* l, const tb2_orca_params* p, const float* pos, const float* vel,
                      const double* goal, const double* speed, float* out, void* stream) {
    TB2_REQUIRE(l && p && pos && vel && goal && speed && out, "null argument");
    return simulate_launch<OrcaSim>("orca_simulate", l, *p, {(const float2*)pos, (const float2*)vel,
                                    (const double2*)goal, speed}, (float2*)out, stream);
}

int tb2_sf_sweep(const tb2_layout* l, const tb2_sf_params* p, const double* params, int32_t P, const double* state,
                 const double* truth, int32_t truth_len, double* ade_out, double* fde_out, void* stream) {
    TB2_REQUIRE(l && p && params && state && truth && ade_out && fde_out, "null argument");
    return sweep_values<SfSim>("sf_sweep", l, *p, params, P, {state}, truth, truth_len, ade_out, fde_out, stream);
}

int tb2_sf_sweep_grad(const tb2_layout* l, const tb2_sf_params* p, const double* params, int32_t P, const double* state,
                      const double* truth, int32_t truth_len, double* ade_out, double* fde_out, double* dade_out,
                      double* dfde_out, void* stream) {
    TB2_REQUIRE(l && p && params && state && truth && ade_out && fde_out && dade_out && dfde_out, "null argument");
    return sweep_launch<SfGradSim>("sf_sweep_grad", l, *p, params, P, truth_len, kSfGradMaxScene, stream,
                                   [&](auto packed, int threads, size_t smem, cudaStream_t st) {
        static DynSmemConfig configured;
        return sweep_form(sf_sweep_grad_kernel<decltype(packed)::value>, configured, l->B, threads, smem, st,
                          l->scene_off, SfGradSim::Inputs{state}, params, P, truth, truth_len, ade_out, fde_out, dade_out,
                          dfde_out, l->B, *p);
    });
}

int tb2_orca_sweep(const tb2_layout* l, const tb2_orca_params* p, const float* params, int32_t P, const float* pos,
                   const float* vel, const double* goal, const double* speed, const double* truth, int32_t truth_len,
                   double* ade_out, double* fde_out, void* stream) {
    TB2_REQUIRE(l && p && params && pos && vel && goal && speed && truth && ade_out && fde_out, "null argument");
    return sweep_values<OrcaSim>("orca_sweep", l, *p, params, P, {(const float2*)pos, (const float2*)vel,
                                 (const double2*)goal, speed}, truth, truth_len, ade_out, fde_out, stream);
}

}  // extern "C"
