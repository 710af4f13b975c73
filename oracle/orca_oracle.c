/*
 * orca_oracle.c -- plain-C restatement of the ORCA step the reference drives through the
 * un-vendored `rvo2` package (Python-RVO2 over RVO2 v2.0.x).  TEST INFRASTRUCTURE, NOT PRODUCT.
 * PARITY UNPINNED vs upstream: rvo2 is absent from /root/reference and this image; the reference
 * holds no test for it.  Anchors:
 *   - call contract: /root/reference/trajnetbaselines/classical/orca.py:84-119
 *       PyRVOSimulator(1/20, nDist, 10, tHorizon, 5, radius, 1.5)                 (:90)
 *       addAgent(pos, maxSpeed = 1.3 * speed, velocity = v)                       (:55)
 *       97 x doStep(), positions sampled when count % 8 == 0                      (:99-108)
 *       pref-velocity <- goal direction clipped to the initial speed, 0 within 0.05 m (:111-119)
 *       the first doStep runs with RVO2's default pref-velocity (0, 0)
 *   - algorithm: van den Berg, Guy, Lin, Manocha, "Reciprocal n-body collision avoidance"
 *     (ORCA) as published in RVO2 v2.0.x: Agent::computeNewVelocity (agent-agent half-planes,
 *     no obstacles), linearProgram1/2/3, RVO_EPSILON = 1e-5, float arithmetic, neighbour list =
 *     the maxNeighbors closest agents within neighborDist sorted by distance (ties: agent index;
 *     upstream's tie order follows its kd-tree traversal, unknowable without the source).
 * Build: oracle/build_c.py (gcc -O2 -ffp-contract=off).
 */
#include <math.h>
#include <stddef.h>
#include <stdlib.h>

#define ORCA_EPS 0.00001f
#define ORCA_MAX_NEIGH 64

typedef struct { float x, y; } v2;
typedef struct { v2 point, dir; } line_t;

static v2 mk(float x, float y) { v2 r; r.x = x; r.y = y; return r; }
static v2 add(v2 a, v2 b) { return mk(a.x + b.x, a.y + b.y); }
static v2 sub(v2 a, v2 b) { return mk(a.x - b.x, a.y - b.y); }
static v2 mul(float s, v2 a) { return mk(s * a.x, s * a.y); }
static float dot(v2 a, v2 b) { return a.x * b.x + a.y * b.y; }
static float det(v2 a, v2 b) { return a.x * b.y - a.y * b.x; }
static float abssq(v2 a) { return dot(a, a); }
static float sqr(float a) { return a * a; }
static v2 normalize(v2 a) { float l = sqrtf(abssq(a)); return mk(a.x / l, a.y / l); }

static int lp1(const line_t* lines, int line_no, float radius, v2 opt, int dir_opt, v2* result) {
    const float dp = dot(lines[line_no].point, lines[line_no].dir);
    const float disc = sqr(dp) + sqr(radius) - abssq(lines[line_no].point);
    if (disc < 0.0f) return 0;
    const float sq = sqrtf(disc);
    float t_left = -dp - sq, t_right = -dp + sq;
    for (int i = 0; i < line_no; ++i) {
        const float den = det(lines[line_no].dir, lines[i].dir);
        const float num = det(lines[i].dir, sub(lines[line_no].point, lines[i].point));
        if (fabsf(den) <= ORCA_EPS) {
            if (num < 0.0f) return 0;
            continue;
        }
        const float t = num / den;
        if (den >= 0.0f) t_right = fminf(t_right, t); else t_left = fmaxf(t_left, t);
        if (t_left > t_right) return 0;
    }
    if (dir_opt) {
        if (dot(opt, lines[line_no].dir) > 0.0f) *result = add(lines[line_no].point, mul(t_right, lines[line_no].dir));
        else *result = add(lines[line_no].point, mul(t_left, lines[line_no].dir));
    } else {
        const float t = dot(lines[line_no].dir, sub(opt, lines[line_no].point));
        if (t < t_left) *result = add(lines[line_no].point, mul(t_left, lines[line_no].dir));
        else if (t > t_right) *result = add(lines[line_no].point, mul(t_right, lines[line_no].dir));
        else *result = add(lines[line_no].point, mul(t, lines[line_no].dir));
    }
    return 1;
}

static int lp2(const line_t* lines, int n, float radius, v2 opt, int dir_opt, v2* result) {
    if (dir_opt) *result = mul(radius, opt);
    else if (abssq(opt) > sqr(radius)) *result = mul(radius, normalize(opt));
    else *result = opt;
    for (int i = 0; i < n; ++i) {
        if (det(lines[i].dir, sub(lines[i].point, *result)) > 0.0f) {
            const v2 tmp = *result;
            if (!lp1(lines, i, radius, opt, dir_opt, result)) {
                *result = tmp;
                return i;
            }
        }
    }
    return n;
}

static void lp3(const line_t* lines, int n, int begin, float radius, v2* result) {
    float distance = 0.0f;
    line_t proj[ORCA_MAX_NEIGH];
    for (int i = begin; i < n; ++i) {
        if (det(lines[i].dir, sub(lines[i].point, *result)) > distance) {
            int np = 0;
            for (int j = 0; j < i; ++j) {
                line_t l;
                const float d = det(lines[i].dir, lines[j].dir);
                if (fabsf(d) <= ORCA_EPS) {
                    if (dot(lines[i].dir, lines[j].dir) > 0.0f) continue;
                    l.point = mul(0.5f, add(lines[i].point, lines[j].point));
                } else {
                    l.point = add(lines[i].point,
                                  mul(det(lines[j].dir, sub(lines[i].point, lines[j].point)) / d, lines[i].dir));
                }
                l.dir = normalize(sub(lines[j].dir, lines[i].dir));
                proj[np++] = l;
            }
            const v2 tmp = *result;
            if (lp2(proj, np, radius, mk(-lines[i].dir.y, lines[i].dir.x), 1, result) < np) *result = tmp;
            distance = det(lines[i].dir, sub(lines[i].point, *result));
        }
    }
}

/* One scene: n agents, all-pairs neighbour search.
 *   pos, vel   [n][2] float  (initial position / velocity)
 *   goal       [n][2] double, speed [n] double (initial speed; maxSpeed = 1.3 * speed)
 *   out        [n_steps / sample_every][n][2] float
 *   counters   NULL, or [4] int64 counts added to: (agent, step) pairs whose neighbour list is full
 *              (max_neighbors); ORCA lines built by the collision branch (distance <= 2 radius);
 *              linearProgram3 calls; (agent, step) pairs whose preferred velocity is zeroed within
 *              end_range of the goal
 */
int orca_simulate_scene(int n, const float* pos_in, const float* vel_in, const double* goal,
                        const double* speed, float time_step, float neighbor_dist, int max_neighbors,
                        float time_horizon, float radius, double end_range, int n_steps,
                        int sample_every, float* out, long long* counters) {
    if (max_neighbors > ORCA_MAX_NEIGH) return -1;
    v2* pos = (v2*)malloc(sizeof(v2) * n);
    v2* vel = (v2*)malloc(sizeof(v2) * n);
    v2* pref = (v2*)malloc(sizeof(v2) * n);
    v2* newv = (v2*)malloc(sizeof(v2) * n);
    float* maxsp = (float*)malloc(sizeof(float) * n);
    for (int i = 0; i < n; ++i) {
        pos[i] = mk(pos_in[2 * i], pos_in[2 * i + 1]);
        vel[i] = mk(vel_in[2 * i], vel_in[2 * i + 1]);
        pref[i] = mk(0.0f, 0.0f);
        maxsp[i] = (float)(1.3 * speed[i]);
    }
    const float inv_th = 1.0f / time_horizon;
    const float inv_ts = 1.0f / time_step;
    int sample = 0;
    for (int count = 1; count <= n_steps; ++count) {
        for (int a = 0; a < n; ++a) {
            /* neighbours: closest max_neighbors within neighbor_dist, sorted by distance */
            int nb[ORCA_MAX_NEIGH];
            float nd[ORCA_MAX_NEIGH];
            int nn = 0;
            float range_sq = sqr(neighbor_dist);
            for (int b = 0; b < n; ++b) {
                if (b == a) continue;
                const float dsq = abssq(sub(pos[a], pos[b]));
                if (dsq < range_sq) {
                    if (nn < max_neighbors) { nb[nn] = b; nd[nn] = dsq; ++nn; }
                    int i = nn - 1;
                    while (i != 0 && dsq < nd[i - 1]) { nb[i] = nb[i - 1]; nd[i] = nd[i - 1]; --i; }
                    nb[i] = b; nd[i] = dsq;
                    if (nn == max_neighbors) range_sq = nd[nn - 1];
                }
            }
            if (counters && nn == max_neighbors) ++counters[0];
            line_t lines[ORCA_MAX_NEIGH];
            for (int k = 0; k < nn; ++k) {
                const int b = nb[k];
                const v2 rp = sub(pos[b], pos[a]);
                const v2 rv = sub(vel[a], vel[b]);
                const float dsq = abssq(rp);
                const float cr = radius + radius;
                const float crsq = sqr(cr);
                line_t l;
                v2 u;
                if (dsq > crsq) {
                    const v2 w = sub(rv, mul(inv_th, rp));
                    const float wsq = abssq(w);
                    const float dp1 = dot(w, rp);
                    if (dp1 < 0.0f && sqr(dp1) > crsq * wsq) {
                        const float wl = sqrtf(wsq);
                        const v2 uw = mk(w.x / wl, w.y / wl);
                        l.dir = mk(uw.y, -uw.x);
                        u = mul(cr * inv_th - wl, uw);
                    } else {
                        const float leg = sqrtf(dsq - crsq);
                        if (det(rp, w) > 0.0f) {
                            l.dir = mk((rp.x * leg - rp.y * cr) / dsq, (rp.x * cr + rp.y * leg) / dsq);
                        } else {
                            l.dir = mk(-(rp.x * leg + rp.y * cr) / dsq, -(-rp.x * cr + rp.y * leg) / dsq);
                        }
                        const float dp2 = dot(rv, l.dir);
                        u = sub(mul(dp2, l.dir), rv);
                    }
                } else {
                    if (counters) ++counters[1];
                    const v2 w = sub(rv, mul(inv_ts, rp));
                    const float wl = sqrtf(abssq(w));
                    const v2 uw = mk(w.x / wl, w.y / wl);
                    l.dir = mk(uw.y, -uw.x);
                    u = mul(cr * inv_ts - wl, uw);
                }
                l.point = add(vel[a], mul(0.5f, u));
                lines[k] = l;
            }
            v2 res;
            const int fail = lp2(lines, nn, maxsp[a], pref[a], 0, &res);
            if (fail < nn) {
                if (counters) ++counters[2];
                lp3(lines, nn, fail, maxsp[a], &res);
            }
            newv[a] = res;
        }
        for (int a = 0; a < n; ++a) {
            vel[a] = newv[a];
            pos[a] = add(pos[a], mul(time_step, vel[a]));
        }
        if (count % sample_every == 0) {
            for (int a = 0; a < n; ++a) {
                out[((size_t)sample * n + a) * 2 + 0] = pos[a].x;
                out[((size_t)sample * n + a) * 2 + 1] = pos[a].y;
            }
            ++sample;
        }
        /* orca.py:111-119, evaluated in double like the reference's numpy code */
        for (int a = 0; a < n; ++a) {
            const double dx = goal[2 * a] - (double)pos[a].x, dy = goal[2 * a + 1] - (double)pos[a].y;
            const double dist = sqrt(dx * dx + dy * dy);
            if (dist < end_range) {
                if (counters) ++counters[3];
                pref[a] = mk(0.0f, 0.0f);
            } else if (dist > speed[a]) {
                pref[a] = mk((float)(speed[a] * dx / dist), (float)(speed[a] * dy / dist));
            } else {
                pref[a] = mk((float)dx, (float)dy);
            }
        }
    }
    free(pos); free(vel); free(pref); free(newv); free(maxsp);
    return 0;
}
