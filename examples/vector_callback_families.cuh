// vector_callback_families.cuh -- USER RHS families that carry their own state-dependent event (not part of the library):
// the conditions and the affect of the reference's VectorContinuousCallback(condition, affect!, NC), compiled into the family
// struct with the derivatives the adjoint needs (csrc/family_plugin.inc, B200ADJ_FAMILY_HAS_EVENTS):
//   condition(u, p, t, out)                 out[c] = g_c(u, p, t)
//   condition_grad(c, u, p, t, gu, gp)      gu = dg_c/du, gp = dg_c/dp, returns dg_c/dt
//   affect(ev, um, p, up)                   ev[c] = +1 / -1 for a condition that crossed upwards / downwards, 0 otherwise
//   affect_vjp(ev, um, p, l, lu, lp)        lu = (d affect/du)' l, lp = (d affect/dp)' l
// Build + register one of them:
//   python -m scimlsensitivity_jl_b200.family_plugin examples/vector_callback_families.cuh ProjectileWall projectile --events
#pragma once
#include <math.h>

#include "families.cuh"

// u = [x, vx, y, vy]: x' = vx, vx' = -p1, y' = vy, vy' = 0 (test/Callbacks2/vector_continuous_callbacks.jl:10-16), p = [g, e]
struct ProjectileFlight {
    static constexpr int D = 4, P = 2, M = 0;
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) { du[0] = u[1]; du[1] = -p[0]; du[2] = u[3]; du[3] = T(0); }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) { dl[0] = T(0); dl[1] = l[0]; dl[2] = T(0); dl[3] = l[2]; }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) { dg[0] = -l[1]; dg[1] = T(0); }
};

// "callback with linear affect" (:78-99): the floor x = 0 and the wall y = 10, the condition of the wall non-linear in u;
// the velocity of the condition that fired is reflected with restitution p[1]
struct ProjectileWall : ProjectileFlight {
    static constexpr int NC = 2;
    __device__ __forceinline__ static void condition(const double* u, const double* p, double t, double* out) {
        out[0] = u[0];
        out[1] = (u[2] - 10.0) * u[2];
    }
    __device__ __forceinline__ static double condition_grad(int c, const double* u, const double* p, double t, double* gu, double* gp) {
        gu[0] = c == 0 ? 1.0 : 0.0; gu[1] = 0.0; gu[2] = c == 1 ? 2.0 * u[2] - 10.0 : 0.0; gu[3] = 0.0;
        gp[0] = 0.0; gp[1] = 0.0;
        return 0.0;
    }
    __device__ __forceinline__ static void affect(const int* ev, const double* um, const double* p, double* up) {
        up[0] = um[0]; up[1] = ev[0] ? -p[1] * um[1] : um[1];
        up[2] = um[2]; up[3] = ev[1] ? -p[1] * um[3] : um[3];
    }
    __device__ __forceinline__ static void affect_vjp(const int* ev, const double* um, const double* p, const double* l, double* lu, double* lp) {
        lu[0] = l[0]; lu[1] = ev[0] ? -p[1] * l[1] : l[1];
        lu[2] = l[2]; lu[3] = ev[1] ? -p[1] * l[3] : l[3];
        lp[0] = 0.0; lp[1] = (ev[0] ? -um[1] * l[1] : 0.0) + (ev[1] ? -um[3] * l[3] : 0.0);
    }
};

// "condition that depends on time only" (:100-117): sin t and cos t, every event resets u to [0.5, 1, 0, 0]
struct ClockReset : ProjectileFlight {
    static constexpr int NC = 2;
    __device__ __forceinline__ static void condition(const double* u, const double* p, double t, double* out) { out[0] = sin(t); out[1] = cos(t); }
    __device__ __forceinline__ static double condition_grad(int c, const double* u, const double* p, double t, double* gu, double* gp) {
        for (int j = 0; j < 4; j++) gu[j] = 0.0;
        gp[0] = 0.0; gp[1] = 0.0;
        return c == 0 ? cos(t) : -sin(t);
    }
    __device__ __forceinline__ static void affect(const int* ev, const double* um, const double* p, double* up) {
        up[0] = 0.5; up[1] = 1.0; up[2] = 0.0; up[3] = 0.0;
    }
    __device__ __forceinline__ static void affect_vjp(const int* ev, const double* um, const double* p, const double* l, double* lu, double* lp) {
        for (int j = 0; j < 4; j++) lu[j] = 0.0;
        lp[0] = 0.0; lp[1] = 0.0;
    }
};

// u = [x, y, vx, vy]: x' = vx, y' = vy, vx' = vy' = 0 (:128-134), p = [unused]
struct PlaneFlight {
    static constexpr int D = 4, P = 1, M = 0;
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) { du[0] = u[2]; du[1] = u[3]; du[2] = T(0); du[3] = T(0); }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) { dl[0] = T(0); dl[1] = T(0); dl[2] = l[0]; dl[3] = l[1]; }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) { dg[0] = T(0); }
};

// "structural simultaneous fire" (:118-168): u[0] and 2 u[0] always fire together; the coupled affect vy <- vx, vx <- -vx
struct TiedWalls : PlaneFlight {
    static constexpr int NC = 2;
    __device__ __forceinline__ static void condition(const double* u, const double* p, double t, double* out) { out[0] = u[0]; out[1] = 2.0 * u[0]; }
    __device__ __forceinline__ static double condition_grad(int c, const double* u, const double* p, double t, double* gu, double* gp) {
        gu[0] = c == 0 ? 1.0 : 2.0; gu[1] = 0.0; gu[2] = 0.0; gu[3] = 0.0;
        gp[0] = 0.0;
        return 0.0;
    }
    __device__ __forceinline__ static void affect(const int* ev, const double* um, const double* p, double* up) {
        up[0] = um[0]; up[1] = um[1]; up[3] = um[2]; up[2] = -um[2];
    }
    __device__ __forceinline__ static void affect_vjp(const int* ev, const double* um, const double* p, const double* l, double* lu, double* lp) {
        lu[0] = l[0]; lu[1] = l[1]; lu[2] = l[3] - l[2]; lu[3] = 0.0;
        lp[0] = 0.0;
    }
};

// "corner trap" (:169-236): the walls x = 0 and y = 0; both at once stop the motion, one alone reflects its velocity
struct CornerWalls : PlaneFlight {
    static constexpr int NC = 2;
    __device__ __forceinline__ static void condition(const double* u, const double* p, double t, double* out) { out[0] = u[0]; out[1] = u[1]; }
    __device__ __forceinline__ static double condition_grad(int c, const double* u, const double* p, double t, double* gu, double* gp) {
        gu[0] = c == 0 ? 1.0 : 0.0; gu[1] = c == 1 ? 1.0 : 0.0; gu[2] = 0.0; gu[3] = 0.0;
        gp[0] = 0.0;
        return 0.0;
    }
    __device__ __forceinline__ static void affect(const int* ev, const double* um, const double* p, double* up) {
        const bool both = ev[0] && ev[1];
        up[0] = um[0]; up[1] = um[1];
        up[2] = both ? 0.0 : (ev[0] ? -um[2] : um[2]);
        up[3] = both ? 0.0 : (ev[1] ? -um[3] : um[3]);
    }
    __device__ __forceinline__ static void affect_vjp(const int* ev, const double* um, const double* p, const double* l, double* lu, double* lp) {
        const bool both = ev[0] && ev[1];
        lu[0] = l[0]; lu[1] = l[1];
        lu[2] = both ? 0.0 : (ev[0] ? -l[2] : l[2]);
        lu[3] = both ? 0.0 : (ev[1] ? -l[3] : l[3]);
        lp[0] = 0.0;
    }
};

// the built-in bouncing ball with its named event as family conditions: x crosses 0 downwards, v <- -p[1] v
struct BallEvents : b200adj::BouncingBall {
    static constexpr int NC = 1;
    __device__ __forceinline__ static void condition(const double* u, const double* p, double t, double* out) { out[0] = u[0]; }
    __device__ __forceinline__ static double condition_grad(int c, const double* u, const double* p, double t, double* gu, double* gp) {
        gu[0] = 1.0; gu[1] = 0.0; gp[0] = 0.0; gp[1] = 0.0;
        return 0.0;
    }
    __device__ __forceinline__ static void affect(const int* ev, const double* um, const double* p, double* up) { up[0] = um[0]; up[1] = -p[1] * um[1]; }
    __device__ __forceinline__ static void affect_vjp(const int* ev, const double* um, const double* p, const double* l, double* lu, double* lp) {
        lu[0] = l[0]; lu[1] = -p[1] * l[1];
        lp[0] = 0.0; lp[1] = -um[1] * l[1];
    }
};

// the named callback of the built-in relax family (test/Callbacks2/continuous_callbacks.jl:317-345): condition u - 3/4 p[0],
// affect u += p[1], both directions
struct RelaxEvents : b200adj::Relax {
    static constexpr int NC = 1;
    __device__ __forceinline__ static void condition(const double* u, const double* p, double t, double* out) { out[0] = u[0] - 0.75 * p[0]; }
    __device__ __forceinline__ static double condition_grad(int c, const double* u, const double* p, double t, double* gu, double* gp) {
        gu[0] = 1.0; gp[0] = -0.75; gp[1] = 0.0;
        return 0.0;
    }
    __device__ __forceinline__ static void affect(const int* ev, const double* um, const double* p, double* up) { up[0] = um[0] + p[1]; }
    __device__ __forceinline__ static void affect_vjp(const int* ev, const double* um, const double* p, const double* l, double* lu, double* lp) {
        lu[0] = l[0]; lp[0] = 0.0; lp[1] = l[0];
    }
};

// van der Pol u0' = u1, u1' = p0 (1 - u0^2) u1 - p1 u0 with a ring event: when |u| grows through the radius p2 the state
// is halved.  A non-polynomial flow with a condition that depends on a parameter.
struct VanDerPolRing {
    static constexpr int D = 2, P = 3, M = 0, NC = 1;
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) {
        du[0] = u[1];
        du[1] = p[0] * (1 - u[0] * u[0]) * u[1] - p[1] * u[0];
    }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) {
        dl[0] = (-2 * p[0] * u[0] * u[1] - p[1]) * l[1];
        dl[1] = l[0] + p[0] * (1 - u[0] * u[0]) * l[1];
    }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) {
        dg[0] = (1 - u[0] * u[0]) * u[1] * l[1];
        dg[1] = -u[0] * l[1];
        dg[2] = T(0);
    }
    __device__ __forceinline__ static void condition(const double* u, const double* p, double t, double* out) { out[0] = u[0] * u[0] + u[1] * u[1] - p[2] * p[2]; }
    __device__ __forceinline__ static double condition_grad(int c, const double* u, const double* p, double t, double* gu, double* gp) {
        gu[0] = 2.0 * u[0]; gu[1] = 2.0 * u[1];
        gp[0] = 0.0; gp[1] = 0.0; gp[2] = -2.0 * p[2];
        return 0.0;
    }
    __device__ __forceinline__ static void affect(const int* ev, const double* um, const double* p, double* up) { up[0] = 0.5 * um[0]; up[1] = 0.5 * um[1]; }
    __device__ __forceinline__ static void affect_vjp(const int* ev, const double* um, const double* p, const double* l, double* lu, double* lp) {
        lu[0] = 0.5 * l[0]; lu[1] = 0.5 * l[1];
        lp[0] = 0.0; lp[1] = 0.0; lp[2] = 0.0;
    }
};
