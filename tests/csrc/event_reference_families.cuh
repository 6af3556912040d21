// event_reference_families.cuh -- test families for the device VectorContinuousCallback (B200ADJ_FAMILY_HAS_EVENTS), each
// built so that its closed form or 40-digit reference pins particular terms of the event-time correction of the reverse
// kernel (tsit5_adaptive.cuh, t5a_reverse_kernel, FE branch):
//   lam- = mu_u - dg/du (w / den),  dG/dp += mu_p - dg/dp (w / den),  den = dg/du . f(u-) + dg/dt
// tests/test_gpu_family_event_references.py builds them into plug-ins and holds their references.
//   MovingWall       NC = 1: dg/dt != 0, dg/dp on two parameters, an affect that depends on two parameters
//   Gates8           NC = 8: the full 16-bit event word, a direction per condition, staggered / tied / one-ulp-apart crossings
//   GatedOscillator  NC = 2: a non-polynomial flow, a condition in u, p and t, a condition non-linear in u, and an affect
//                    whose Jacobian is non-diagonal and depends on the state and on p
#pragma once
#include <math.h>

#include "families.cuh"

// u = [x, v]: x' = v, v' = -p0.  The wall x = p1 + p2 t moves at speed p2; the ball bounces off it with restitution p3
// relative to the wall, v+ = p2 - p3 (v- - p2).  Quadratic flight: Tsit5 and its interpolant are exact.
struct MovingWall {
    static constexpr int D = 2, P = 4, M = 0, NC = 1;
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) { du[0] = u[1]; du[1] = -p[0]; }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) { dl[0] = T(0); dl[1] = l[0]; }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) {
        dg[0] = -l[1]; dg[1] = T(0); dg[2] = T(0); dg[3] = T(0);
    }
    __device__ __forceinline__ static void condition(const double* u, const double* p, double t, double* out) { out[0] = u[0] - p[1] - p[2] * t; }
    __device__ __forceinline__ static double condition_grad(int c, const double* u, const double* p, double t, double* gu, double* gp) {
        gu[0] = 1.0; gu[1] = 0.0;
        gp[0] = 0.0; gp[1] = -1.0; gp[2] = -t; gp[3] = 0.0;
        return -p[2];
    }
    __device__ __forceinline__ static void affect(const int* ev, const double* um, const double* p, double* up) {
        up[0] = um[0]; up[1] = p[2] - p[3] * (um[1] - p[2]);
    }
    __device__ __forceinline__ static void affect_vjp(const int* ev, const double* um, const double* p, const double* l, double* lu, double* lp) {
        lu[0] = l[0]; lu[1] = -p[3] * l[1];
        lp[0] = 0.0; lp[1] = 0.0; lp[2] = (1.0 + p[3]) * l[1]; lp[3] = -(um[1] - p[2]) * l[1];
    }
};

// u = [x, v]: a particle at constant velocity between the walls x = 1 (c0, v <- -p0 v) and x = 0 (c1, v <- -p1 v), through
// six gates x = GATE_LEVEL[c] (c2..c7, v <- p_c v).  The gains commute, so gates that fire together and gates that fire one
// after the other leave the same state.  c2 / c3 are 1e-7 apart (one sample interval, two roots), c4 / c5 share a level
// (directions -1 and 0 in the tests: downwards both fire, upwards only c5), c6 / c7 are one ulp apart.
struct Gates8 {
    static constexpr int D = 2, P = 8, M = 0, NC = 8;
    __device__ __forceinline__ static double level(int c) {
        switch (c) {
            case 0: return 1.0;
            case 1: return 0.0;
            case 2: return 0.3;
            case 3: return 0.3000001;
            case 4: case 5: return 0.55;
            case 6: return 0.8;
            default: return 0x1.999999999999bp-1;        // nextafter(0.8, 1): 0.8 is 0x1.999999999999ap-1
        }
    }
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) { du[0] = u[1]; du[1] = T(0); }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) { dl[0] = T(0); dl[1] = l[0]; }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) {
        for (int q = 0; q < P; q++) dg[q] = T(0);
    }
    __device__ __forceinline__ static void condition(const double* u, const double* p, double t, double* out) {
        for (int c = 0; c < NC; c++) out[c] = u[0] - level(c);
    }
    __device__ __forceinline__ static double condition_grad(int c, const double* u, const double* p, double t, double* gu, double* gp) {
        gu[0] = 1.0; gu[1] = 0.0;
        for (int q = 0; q < P; q++) gp[q] = 0.0;
        return 0.0;
    }
    // the velocity's gain from the conditions that fired (walls reflect)
    __device__ __forceinline__ static double gain(const int* ev, const double* p) {
        double k = 1.0;
        for (int c = 0; c < NC; c++) if (ev[c]) k *= c < 2 ? -p[c] : p[c];
        return k;
    }
    __device__ __forceinline__ static void affect(const int* ev, const double* um, const double* p, double* up) {
        up[0] = um[0]; up[1] = gain(ev, p) * um[1];
    }
    __device__ __forceinline__ static void affect_vjp(const int* ev, const double* um, const double* p, const double* l, double* lu, double* lp) {
        const double k = gain(ev, p);
        lu[0] = l[0]; lu[1] = k * l[1];
        for (int q = 0; q < P; q++) lp[q] = ev[q] ? k / p[q] * um[1] * l[1] : 0.0;     // d(k v)/dp_q = k / p_q v
    }
};

// u' = A(p) u with A = [[-p0, p1], [-p1, -p0]] (a damped rotation).  c0: u0 - p2 cos t (both directions; depends on u, p
// and t); c1: |u|^2 - p3^2 (the ring, non-linear in u).  Affect: c0 fired -> u1 <- u1 - u0 u1 / 2 + p4 u0; then c1 fired ->
// u <- 1.25 u (the state is pushed back out of the ring).
struct GatedOscillator {
    static constexpr int D = 2, P = 5, M = 0, NC = 2;
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) {
        du[0] = -p[0] * u[0] + p[1] * u[1];
        du[1] = -p[1] * u[0] - p[0] * u[1];
    }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) {
        dl[0] = -p[0] * l[0] - p[1] * l[1];
        dl[1] = p[1] * l[0] - p[0] * l[1];
    }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) {
        dg[0] = -u[0] * l[0] - u[1] * l[1];
        dg[1] = u[1] * l[0] - u[0] * l[1];
        dg[2] = T(0); dg[3] = T(0); dg[4] = T(0);
    }
    __device__ __forceinline__ static void condition(const double* u, const double* p, double t, double* out) {
        out[0] = u[0] - p[2] * cos(t);
        out[1] = u[0] * u[0] + u[1] * u[1] - p[3] * p[3];
    }
    __device__ __forceinline__ static double condition_grad(int c, const double* u, const double* p, double t, double* gu, double* gp) {
        for (int q = 0; q < P; q++) gp[q] = 0.0;
        if (c == 0) {
            gu[0] = 1.0; gu[1] = 0.0; gp[2] = -cos(t);
            return p[2] * sin(t);
        }
        gu[0] = 2.0 * u[0]; gu[1] = 2.0 * u[1]; gp[3] = -2.0 * p[3];
        return 0.0;
    }
    __device__ __forceinline__ static void affect(const int* ev, const double* um, const double* p, double* up) {
        up[0] = um[0]; up[1] = um[1];
        if (ev[0]) up[1] = um[1] - 0.5 * um[0] * um[1] + p[4] * um[0];
        if (ev[1]) { up[0] *= 1.25; up[1] *= 1.25; }
    }
    __device__ __forceinline__ static void affect_vjp(const int* ev, const double* um, const double* p, const double* l, double* lu, double* lp) {
        const double s = ev[1] ? 1.25 : 1.0;
        const double l0 = s * l[0], l1 = s * l[1];
        for (int q = 0; q < P; q++) lp[q] = 0.0;
        lu[0] = l0; lu[1] = l1;
        if (ev[0]) {          // d(u1 - u0 u1 / 2 + p4 u0) = (p4 - u1 / 2) du0 + (1 - u0 / 2) du1 + u0 dp4
            lu[0] = l0 + (p[4] - 0.5 * um[1]) * l1;
            lu[1] = (1.0 - 0.5 * um[0]) * l1;
            lp[4] = um[0] * l1;
        }
    }
};
