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

#include "common.cuh"

namespace tb2 {

// =========================================================================================
// social force (double precision like upstream numpy)
// =========================================================================================
struct SfScene {
    double* px; double* py; double* vx; double* vy; double* ex; double* ey; double* sp;
};

__device__ __forceinline__ double sf_potential(double rx, double ry, double sb, double ebx, double eby,
                                               double dt, double v0, double sigma) {
    // V(r_ab) = v0 exp(-b / sigma), b = 0.5 sqrt((|r| + |r - dt s_b e_b|)^2 - (dt s_b)^2)
    const double n1 = sqrt(rx * rx + ry * ry);
    const double qx = rx - dt * sb * ebx, qy = ry - dt * sb * eby;
    const double n2 = sqrt(qx * qx + qy * qy);
    const double s = n1 + n2;
    const double in_sqrt = s * s - (dt * sb) * (dt * sb);
    const double b = 0.5 * sqrt(in_sqrt);
    return v0 * exp(-b / sigma);
}

// One pedestrian of a social-force rollout: position, velocity, destination, initial and maximum speed
// (Simulator.__init__: initial_speeds, max_speeds = 1.3 x).
struct SfAgent { double x, y, ux, uy, dx, dy, s0, smax; };

__device__ __forceinline__ SfAgent sf_agent_init(const double* st) {
    SfAgent g;
    g.x = st[0]; g.y = st[1]; g.ux = st[2]; g.uy = st[3]; g.dx = st[4]; g.dy = st[5];
    g.s0 = sqrt(g.ux * g.ux + g.uy * g.uy);
    g.smax = 1.3 * g.s0;
    return g;
}

__device__ __forceinline__ double sf_cosphi() { return cos(200.0 / 2.0 / 180.0 * 3.141592653589793); }   // FieldOfView(twophi=200)

// First half of a step: the desired direction (NaN at the destination, as upstream), published with the state for the
// neighbour loop of every pedestrian of the scene.
__device__ __forceinline__ void sf_publish(const SfAgent& g, const SfScene& sc, int a, double& eax, double& eay) {
    const double gx = g.dx - g.x, gy = g.dy - g.y;
    const double gn = sqrt(gx * gx + gy * gy);
    eax = gx / gn; eay = gy / gn;
    sc.px[a] = g.x; sc.py[a] = g.y; sc.vx[a] = g.ux; sc.vy[a] = g.uy; sc.ex[a] = eax; sc.ey[a] = eay;
    sc.sp[a] = sqrt(g.ux * g.ux + g.uy * g.uy);
}

// Second half: driving force + pairwise repulsion over b = 0 .. n-1 in index order, speed clip, position update.
__device__ __forceinline__ void sf_advance(SfAgent& g, const SfScene& sc, int a, int n, double eax, double eay,
                                           double dt, double tau, double v0, double sigma, double cosphi) {
    const double fd = 1e-3;
    double Fx = 1.0 / tau * (g.s0 * eax - g.ux);
    double Fy = 1.0 / tau * (g.s0 * eay - g.uy);
    double sumx = 0.0, sumy = 0.0;
    for (int b = 0; b < n; ++b) {
        double fx = 0.0, fy = 0.0, w = 0.0;
        if (b != a) {
            const double rx = g.x - sc.px[b], ry = g.y - sc.py[b];
            const double sb = sc.sp[b], ebx = sc.ex[b], eby = sc.ey[b];
            const double v = sf_potential(rx, ry, sb, ebx, eby, dt, v0, sigma);
            const double dvdx = (sf_potential(rx + fd, ry, sb, ebx, eby, dt, v0, sigma) - v) / fd;
            const double dvdy = (sf_potential(rx, ry + fd, sb, ebx, eby, dt, v0, sigma) - v) / fd;
            fx = -1.0 * dvdx; fy = -1.0 * dvdy;               // f_ab = -grad V
            const double gx = -fx, gy = -fy;                  // w(e, -f_ab)
            const bool in_sight = (eax * gx + eay * gy) > sqrt(gx * gx + gy * gy) * cosphi;
            w = in_sight ? 1.0 : 0.5;
        }
        sumx += w * fx;
        sumy += w * fy;
    }
    Fx += sumx; Fy += sumy;
    const double wx = g.ux + dt * Fx, wy = g.uy + dt * Fy;
    const double wn = sqrt(wx * wx + wy * wy);
    const double q = g.smax / wn;
    const double factor = isnan(q) ? q : (q < 1.0 ? q : 1.0);       // numpy.minimum(1, q)
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

struct SfSim {
    using Params = tb2_sf_params;
    using Setting = double;                    // tau, v0, sigma
    using Agent = SfAgent;
    using Scene = SfScene;
    using Handoff = double2;                   // phase 1 -> phase 2: the desired direction
    using Pos = double2;
    struct Inputs { const double* state; };
    struct Consts { double dt, tau, v0, sigma, cosphi; };
    static constexpr size_t kPedBytes = 7 * sizeof(double);
    static constexpr int kSampleOffset = 0;    // sample after step k = 0 .. n_steps - 1 when k % sample_every == 0

    __device__ static Agent agent(const Inputs& in, int row) { return sf_agent_init(in.state + (size_t)row * 6); }
    __device__ static Consts consts(const Params& p, const Setting* row) {
        return {(double)p.delta_t, row ? row[0] : (double)p.tau, row ? row[1] : (double)p.v0,
                row ? row[2] : (double)p.sigma, sf_cosphi()};
    }
    // The scene arrays from pedestrian slot `first` on, each `stride` long.
    __device__ static Scene scene(void* arrays, size_t first, int stride) {
        double* px = static_cast<double*>(arrays) + first * 7;
        return {px, px + stride, px + 2 * stride, px + 3 * stride, px + 4 * stride, px + 5 * stride, px + 6 * stride};
    }
    template <bool kWarp>
    __device__ static void prologue(const Agent&, const Scene&, int, bool) {}
    __device__ static Handoff phase1(const Agent& g, const Consts&, const Scene& sc, int a, int) {
        double2 e;
        sf_publish(g, sc, a, e.x, e.y);
        return e;
    }
    __device__ static void phase2(Agent& g, const Consts& c, const Scene& sc, int a, int n, Handoff e) {
        sf_advance(g, sc, a, n, e.x, e.y, c.dt, c.tau, c.v0, c.sigma, c.cosphi);
    }
    __device__ static Pos position(const Agent& g) { return make_double2(g.x, g.y); }

    static int check(const Params&) { return TB2_OK; }
    static int check_setting(const Setting* s) {
        TB2_REQUIRE(s[0] > 0.0 && s[2] > 0.0, "tau and sigma must be > 0");
        return TB2_OK;
    }
};

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

static int sweep_counts(const tb2_layout* l, int P, int T, int n_samples) {
    TB2_REQUIRE(l->B >= 1, "no scenes");
    TB2_REQUIRE(P >= 1, "P < 1 settings");
    TB2_REQUIRE((int64_t)P * l->B < ((int64_t)1 << 31), "P x B >= 2^31");
    TB2_REQUIRE(l->n_max <= 1024, "scene larger than 1024 pedestrians");
    TB2_REQUIRE(n_samples >= 1 && n_samples <= 1024, "sample count must be in [1, 1024]");
    TB2_REQUIRE(T >= n_samples, "truth shorter than the sample count");
    return TB2_OK;
}

// Checks the call, then launches both forms over every scene; each CTA keeps only the scenes of its form (packed:
// n <= 32, CTA: n > 32).
template <class Sim>
static int sweep_launch(const char* name, const tb2_layout* l, const typename Sim::Params& p,
                        const typename Sim::Setting* params, int P, typename Sim::Inputs in, const double* truth, int T,
                        double* ade, double* fde, void* stream) {
    int rc = check_rollout<Sim>(p);
    if (rc != TB2_OK) return rc;
    const int n_samples = sample_count<Sim>(p.n_steps, p.sample_every);
    rc = sweep_counts(l, P, T, n_samples);
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
    sweep_kernel<Sim, true><<<l->B, 32 * warps, truth_bytes + (size_t)32 * warps * Sim::kPedBytes, st>>>(
        l->scene_off, in, params, P, truth, T, ade, fde, l->B, p);
    TB2_LAUNCH_CHECK();
    if (l->n_max > 32) {
        const int threads = (l->n_max + 31) / 32 * 32;
        const size_t smem = truth_bytes + (size_t)l->n_max * Sim::kPedBytes;
        static DynSmemConfig configured;
        TB2_CHECK_CUDA(configured.ensure(sweep_kernel<Sim, false>, smem, 48 * 1024));
        sweep_kernel<Sim, false><<<l->B, threads, smem, st>>>(l->scene_off, in, params, P, truth, T, ade, fde, l->B, p);
        TB2_LAUNCH_CHECK();
    }
    return TB2_OK;
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
    return sweep_launch<SfSim>("sf_sweep", l, *p, params, P, {state}, truth, truth_len, ade_out, fde_out, stream);
}

int tb2_orca_sweep(const tb2_layout* l, const tb2_orca_params* p, const float* params, int32_t P, const float* pos,
                   const float* vel, const double* goal, const double* speed, const double* truth, int32_t truth_len,
                   double* ade_out, double* fde_out, void* stream) {
    TB2_REQUIRE(l && p && params && pos && vel && goal && speed && truth && ade_out && fde_out, "null argument");
    return sweep_launch<OrcaSim>("orca_sweep", l, *p, params, P, {(const float2*)pos, (const float2*)vel,
                                 (const double2*)goal, speed}, truth, truth_len, ade_out, fde_out, stream);
}

}  // extern "C"
