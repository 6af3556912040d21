// quadgk.cuh -- warp-cooperative adaptive Gauss-Kronrod (7,15) quadrature: QuadGK.jl's adapt loop (bisect the largest-error
// segment until E <= max(atol, rtol |I|), running totals updated incrementally) with ONE WARP PER MEMBER.  Used by the
// QuadratureAdjoint kernels of all three ODE steppers (src/quadrature_adjoint.jl:486-502 integrand, :537-616 interval loop).
//
// What a bisection costs here (round-2 redesign; the first version spent 98 of 143 ms of config C3 in dependent global
// loads: a 12-level binary search per node in each dense solution and a binary heap sifted by lane 0):
//   * 30 of the 32 lanes evaluate the 2 x 15 Kronrod nodes of the two halves; lanes 15 / 31 look up the bisection point.
//   * dense-solution lookup: every segment carries the index BRACKETS of both dense solutions (inherited from its parent
//     and narrowed at the bisection point), so a node is located among <= 32 knots that the warp fetches with ONE coalesced
//     round of loads and searches with shuffles (wider brackets: 32 strided samples, then a short per-lane search);
//   * priority queue: segments never move.  Keys (segment errors) sit in a flat per-warp array; the maxima of its
//     32-key blocks live in shared memory; arg-max = scan of the block maxima (shared memory) + one coalesced 256 B load of
//     the winning block + shuffles.  Ties resolve to the lowest segment index, as the oracle's linear scan does.
//   * scratch is per RESIDENT warp (persistent grid-stride kernel), not per member.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200adj {

__device__ const double XGK[8] = {0.991455371120812639206854697526329, 0.949107912342758524526189684047851,
    0.864864423359769072789712788640926, 0.741531185599394439863864773280788, 0.586087235467691130294144838258730,
    0.405845151377397166906606412076961, 0.207784955007898467600689403773245, 0.0};
__device__ const double WGK[8] = {0.022935322010529224963732008058970, 0.063092092629978553290700663189204,
    0.104790010322250183839876322541518, 0.140653259715525918745189590510238, 0.169004726639267902826583426598550,
    0.190350578064785409913256402421014, 0.204432940075298892414161999234649, 0.209482141084727828012999174891714};
__device__ const double WG[4] = {0.129484966168869693270611432679082, 0.279705391489276667901467771423780,
    0.381830050505118944950369775488975, 0.417959183673469387755102040816327};

constexpr int QUAD_WARPS = 4;                 // warps (members in flight) per block
constexpr int QUAD_BLOCKS_PER_SM = 6;         // persistent grid = min(ceil(N / 4), n_SM * 6)
template <int P> __host__ __device__ constexpr int quad_segw() { return ((P + 4 + 3) / 4) * 4; }      // doubles per segment record (32 B multiple)
// bytes of segment scratch one resident warp needs
template <int P> __host__ __device__ constexpr size_t quad_scratch_bytes(int maxseg) { return (size_t)maxseg * (quad_segw<P>() + 1) * sizeof(double); }

// record widths are padded to whole 32 B sectors
__host__ __device__ constexpr int quad_pad(int n) { return ((n + 3) / 4) * 4; }

// Member-major copy of the forward dense solution (member-minor ft[MAXS+1][N], fu[MAXS+1][D][N], fk[MAXS][NK][D][N], written
// coalesced by the thread-per-member solvers) for the warp-per-member quadrature kernel: ftT[N][MAXS+1],
// frecT[N][MAXS][pad(D + NK D + 3)] = (u[D], k[NK][D], t_a, h, 1/h).  Thread (j, i): i fastest => coalesced reads.
template <int UNUSED = 0>
__global__ void quad_transpose_fwd_kernel(const double* ft, const double* fu, const double* fk, const int32_t* fn, double* ftT, double* frecT,
                                          int64_t N, int maxs, int D, int NK) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int n = fn[i];
    for (int j = blockIdx.y; j <= n; j += gridDim.y) {
    const double ta = ft[(int64_t)j * N + i];
    ftT[i * (maxs + 1) + j] = ta;
    if (j == n) break;
    const int FWP = quad_pad(D + NK * D + 3);
    double* r = frecT + (i * maxs + j) * FWP;
    for (int c = 0; c < D; c++) r[c] = fu[((int64_t)j * D + c) * N + i];
    for (int s = 0; s < NK; s++)
        for (int c = 0; c < D; c++) r[(1 + s) * D + c] = fk[(((int64_t)j * NK + s) * D + c) * N + i];
    const double h = ft[(int64_t)(j + 1) * N + i] - ta;
    r[D + NK * D] = ta; r[D + NK * D + 1] = h; r[D + NK * D + 2] = 1.0 / h;
    }
}

// index brackets of a segment in the forward (flo..fhi) and reverse (rlo..rhi) dense solutions
struct QuadBracket { int flo, fhi, rlo, rhi; };

// number of entries of an ASCENDING knot sequence that are < t, for knots held one per lane (lane j holds knot j,
// j < cnt <= 32); all lanes take part.  Short sequences (the common case: a segment spans a few steps) are scanned,
// longer ones searched by bisection over the lanes.
__device__ __forceinline__ int lanes_count_less(double knot, int cnt, double t) {
    int pos = 0;
    if (cnt <= 6) {
        for (int k = 0; k < cnt; k++) pos += __shfl_sync(0xffffffffu, knot, k) < t ? 1 : 0;      // monotone: a prefix is counted
        return pos;
    }
#pragma unroll
    for (int s = 32; s > 0; s >>= 1) {
        const int probe = pos + s - 1;
        const double v = __shfl_sync(0xffffffffu, knot, probe & 31);
        if (pos + s <= cnt && v < t) pos += s;
    }
    return pos;
}
// same for a DESCENDING sequence: entries > t
__device__ __forceinline__ int lanes_count_greater(double knot, int cnt, double t) {
    int pos = 0;
    if (cnt <= 6) {
        for (int k = 0; k < cnt; k++) pos += __shfl_sync(0xffffffffu, knot, k) > t ? 1 : 0;
        return pos;
    }
#pragma unroll
    for (int s = 32; s > 0; s >>= 1) {
        const int probe = pos + s - 1;
        const double v = __shfl_sync(0xffffffffu, knot, probe & 31);
        if (pos + s <= cnt && v > t) pos += s;
    }
    return pos;
}

// Cooperative location of every lane's t among `cnt` candidate knots first .. first+cnt-1 of a monotone sequence given by
// `knot(j)` (a global load).  ASC: returns #{candidates < t};  !ASC (descending sequence): #{candidates > t}.
template <bool ASC, class KNOT>
__device__ __forceinline__ int coop_count(const KNOT& knot, int first, int cnt, double t, int lane) {
    if (cnt <= 0) return 0;
    if (cnt <= 32) {
        const double kv = lane < cnt ? knot(first + lane) : 0.0;
        return ASC ? lanes_count_less(kv, cnt, t) : lanes_count_greater(kv, cnt, t);
    }
    // wide bracket: 32 strided samples (knot first + (j+1) stride - 1, j = 0..ns-1), then a per-lane search inside one stride
    const int stride = (cnt + 31) >> 5, ns = cnt / stride;          // ns <= 32 full strides
    const double kv = lane < ns ? knot(first + (lane + 1) * stride - 1) : 0.0;
    const int full = ASC ? lanes_count_less(kv, ns, t) : lanes_count_greater(kv, ns, t);     // strides entirely counted
    int lo = full * stride, hi = min(cnt, lo + stride);             // answer = lo + count inside [lo, hi)
    while (lo < hi) {                                               // first index in [lo, hi) whose knot is NOT counted
        const int mid = (lo + hi) >> 1;
        const double v = knot(first + mid);
        if (ASC ? (v < t) : (v > t)) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// warp arg-max of non-negative doubles (masked lanes pass present = false): two integer REDUX on the bit pattern (the order
// of non-negative doubles is the order of their bits) and a ballot; ties resolve to the lowest lane.
__device__ __forceinline__ int warp_argmax_lane(double v, bool present) {
    const int hi = present ? __double2hiint(v) : -1;
    const int mh = __reduce_max_sync(0xffffffffu, hi);
    const unsigned lo = (present && hi == mh) ? (unsigned)__double2loint(v) : 0u;
    const unsigned ml = __reduce_max_sync(0xffffffffu, lo);
    const unsigned b = __ballot_sync(0xffffffffu, present && hi == mh && lo == ml);
    return __ffs(b) - 1;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, off));
    return v;
}

// Gauss-Kronrod (7,15) on the two halves [a0,b0], [a1,b1] of a segment whose bracket is `br`: lanes 0..14 / 16..30 take the
// 15 nodes of the left / right half (node order: lane l -> abscissa sign(l-7) XGK[min(l,14-l)], ascending in t); lanes 15
// and 31 evaluate the integrand's lookups at `tsplit` (the bisection point) so that the children's brackets are known.
// f.eval(t, br, lane, out, &fiv, &riv) is called by ALL lanes (its lookups are warp-cooperative).
// On return EVERY lane of a half holds that half's Kronrod integral Ih[P] and error estimate eh.
template <int P, class F>
__device__ __forceinline__ void gk15_pair(const F& f, const QuadBracket& br, double a0, double b0, double a1, double b1, double tsplit, int lane,
                                          double* Ih, double* eh, int* fsplit, int* rsplit) {
    const int half = lane >> 4, l = lane & 15;
    const double a = half ? a1 : a0, b = half ? b1 : b0;
    const double c = 0.5 * (a + b), hl = 0.5 * (b - a);
    const int j = l < 7 ? l : 14 - l;                      // 0..7 (7 = centre); lane 15: j = -1
    const double x = l < 15 ? (l < 7 ? -XGK[j] : XGK[j]) : 0.0;
    const double t = l < 15 ? c + hl * x : tsplit;
    double w[P], vg[P];
    int fiv, riv;
    f.eval(t, br, lane, w, &fiv, &riv);
    const double wk = l < 15 ? WGK[j] : 0.0, wg = l < 15 ? ((j == 7) ? WG[3] : ((j & 1) ? WG[j >> 1] : 0.0)) : 0.0;
#pragma unroll
    for (int q = 0; q < P; q++) { Ih[q] = l < 15 ? wk * w[q] : 0.0; vg[q] = l < 15 ? wg * w[q] : 0.0; }
#pragma unroll
    for (int q = 0; q < P; q++) {
#pragma unroll
        for (int off = 8; off > 0; off >>= 1) { Ih[q] += __shfl_xor_sync(0xffffffffu, Ih[q], off); vg[q] += __shfl_xor_sync(0xffffffffu, vg[q], off); }
    }
    double e2 = 0;
#pragma unroll
    for (int q = 0; q < P; q++) { Ih[q] *= hl; vg[q] *= hl; e2 += (Ih[q] - vg[q]) * (Ih[q] - vg[q]); }
    *eh = sqrt(e2);
    *fsplit = __shfl_sync(0xffffffffu, fiv, 15); *rsplit = __shfl_sync(0xffffffffu, riv, 15);
}

// per-warp segment store.  Global (owned by this resident warp): seg[maxseg][SEGW] = (a, b, I[P], (flo, fhi), (rlo, rhi)) and
// the keys (segment errors) of the segments >= QUAD_SKEYS.  Shared memory: skey[QUAD_SKEYS] = keys of the first segments (a data
// interval rarely needs more), l1[quad_l1_blocks(maxseg)] = maxima of the 32-key blocks.
constexpr int QUAD_SKEYS = 512;
struct QuadScratch { double* seg; double* key; double* skey; double* l1; int maxseg; };
// block maxima one warp keeps: key maxseg - 1 lies in block (maxseg - 1) >> 5, so a partial last block needs its own entry
__host__ __device__ constexpr int quad_l1_blocks(int maxseg) { return (maxseg + 31) >> 5; }

__device__ __forceinline__ double pack2(int a, int b) { return __longlong_as_double(((long long)(unsigned int)a) | ((long long)b << 32)); }
__device__ __forceinline__ void unpack2(double v, int* a, int* b) { const long long x = __double_as_longlong(v); *a = (int)(unsigned int)(x & 0xffffffffLL); *b = (int)(x >> 32); }

// arg-max of the keys of segments 0 .. nseg-1: block maxima (shared memory), then the winning block's 32 keys.  Ties resolve to
// the lowest segment index, as the oracle's linear scan: lane l scans blocks l, l+32, ... keeping its first maximum, and among
// the lanes that hold the maximum the lowest BLOCK index wins (the lowest lane would prefer block 32 over block 1).
// -> bi = winning block, w = winning segment, ew = its key; kv = this lane's key of block bi (0 past nseg).
struct QuadPick { int bi, w; double ew, kv; };
__device__ __forceinline__ QuadPick quad_queue_argmax(const QuadScratch& q, int nseg, int lane) {
    const int nb = (nseg + 31) >> 5;
    int bi = 0;
    if (nb > 1) {
        double bv = 0.0; int bl = -1;
        for (int bb = lane; bb < nb; bb += 32) { const double v = q.l1[bb]; if (bl < 0 || v > bv) { bv = v; bl = bb; } }
        const int src = warp_argmax_lane(bv, bl >= 0);
        const long long mx = __double_as_longlong(__shfl_sync(0xffffffffu, bv, src));
        bi = __reduce_min_sync(0xffffffffu, (unsigned)((bl >= 0 && __double_as_longlong(bv) == mx) ? bl : 0x7fffffff));
    }
    const int kidx = bi * 32 + lane;
    const double kv = kidx < nseg ? (kidx < QUAD_SKEYS ? q.skey[kidx] : __ldcg(q.key + kidx)) : 0.0;
    const int wl = warp_argmax_lane(kv, kidx < nseg);
    return QuadPick{bi, bi * 32 + wl, __shfl_sync(0xffffffffu, kv, wl), kv};
}

// adaptive quadgk over [a,b] by one warp.  `root` = index bracket of the whole panel.  false = out of segment capacity.
template <int P, class F>
__device__ bool quadgk_warp(const F& f, const QuadBracket& root, double a, double b, double atol, double rtol, double* out, const QuadScratch& q, int lane) {
    static_assert(P <= 12, "a segment record (a, b, I[P], two brackets) is stored by at most 16 lanes of a half warp");
    constexpr int SEGW = quad_segw<P>();
    const int half = lane >> 4, c = lane & 15;             // c: element of the segment record this lane stores
    double Ih[P], Itot[P], eh, Etot;
    int fs, rs;
    gk15_pair<P>(f, root, a, b, a, b, b, lane, Ih, &eh, &fs, &rs);
    {   // segment 0
        double v = c == 0 ? a : c == 1 ? b : c == 2 + P ? pack2(root.flo, root.fhi) : c == 3 + P ? pack2(root.rlo, root.rhi) : 0.0;
#pragma unroll
        for (int k = 0; k < P; k++) if (c == 2 + k) v = Ih[k];
        if (lane < SEGW) q.seg[lane] = v;
        if (lane == 0) { q.skey[0] = eh; q.l1[0] = eh; }
    }
#pragma unroll
    for (int k = 0; k < P; k++) Itot[k] = Ih[k];
    Etot = eh;
    int nseg = 1;
    bool ok = true;
    __syncwarp();
    for (;;) {
        double nI = 0;
#pragma unroll
        for (int k = 0; k < P; k++) nI += Itot[k] * Itot[k];
        nI = sqrt(nI);
        if (Etot <= fmax(atol, rtol * nI)) break;
        if (nseg + 1 > q.maxseg) { ok = false; break; }
        // ---- arg-max of the segment errors ----
        const QuadPick pk = quad_queue_argmax(q, nseg, lane);
        const int bi = pk.bi, w = pk.w;
        const double ew = pk.ew, kv = pk.kv;
        // ---- the segment record (every lane reads the same addresses: broadcast loads) ----
        const double* sr = q.seg + (size_t)w * SEGW;
        const double aw = __ldcg(sr), bw = __ldcg(sr + 1);
        QuadBracket br;
        unpack2(__ldcg(sr + 2 + P), &br.flo, &br.fhi);
        unpack2(__ldcg(sr + 3 + P), &br.rlo, &br.rhi);
        double Iold[P];
#pragma unroll
        for (int k = 0; k < P; k++) Iold[k] = __ldcg(sr + 2 + k);
        const double mid = 0.5 * (aw + bw);
        if (!(mid > fmin(aw, bw) && mid < fmax(aw, bw))) break;
        gk15_pair<P>(f, br, aw, mid, mid, bw, mid, lane, Ih, &eh, &fs, &rs);
        // lanes 0..15 hold the left half's (I, e), lanes 16..31 the right half's
        const double eo = __shfl_xor_sync(0xffffffffu, eh, 16);
        const double el = half ? eo : eh, er = half ? eh : eo;
        Etot += (el + er) - ew;
#pragma unroll
        for (int k = 0; k < P; k++) {
            const double io = __shfl_xor_sync(0xffffffffu, Ih[k], 16);
            Itot[k] += ((half ? io : Ih[k]) + (half ? Ih[k] : io)) - Iold[k];
        }
        // ---- store: w <- left half (lanes 0..), nseg <- right half (lanes 16..); children inherit the bracket narrowed at
        //      the bisection point ----
        {
            double v = c == 0 ? (half ? mid : aw) : c == 1 ? (half ? bw : mid)
                     : c == 2 + P ? (half ? pack2(fs, br.fhi) : pack2(br.flo, fs)) : c == 3 + P ? (half ? pack2(br.rlo, rs) : pack2(rs, br.rhi)) : 0.0;
#pragma unroll
            for (int k = 0; k < P; k++) if (c == 2 + k) v = Ih[k];
            if (c < SEGW) q.seg[(size_t)(half ? nseg : w) * SEGW + c] = v;
        }
        const int bn = nseg >> 5;
        double kn = lane == (w & 31) ? el : kv;
        if (bn == bi && lane == (nseg & 31)) kn = er;
        const double m = warp_max(kn);
        if (lane == 0) {
            if (w < QUAD_SKEYS) q.skey[w] = el; else q.key[w] = el;
            if (nseg < QUAD_SKEYS) q.skey[nseg] = er; else q.key[nseg] = er;
            q.l1[bi] = m;
            if (bn != bi) q.l1[bn] = (nseg & 31) == 0 ? er : fmax(q.l1[bn], er);
        }
        __syncwarp();
        nseg++;
    }
#pragma unroll
    for (int k = 0; k < P; k++) out[k] = Itot[k];
    return ok;
}

// ---- GaussKronrodAdjoint: IntegratingGKSumCallback [UPSTREAM DiffEqCallbacks, restated; gauss_adjoint.jl:820-825].
// After every accepted reverse step the integrand is integrated over [tprev, t] with a Gauss-Kronrod pair of
// ORDER = div(alg_order + 1, 2) Gauss points (Tsit5: G3/K7, Rosenbrock23: G1/K3); if sum|K - G| >= 1e-7 the interval is
// bisected and both halves are integrated (left first), otherwise K joins the running sum.  The recursion is an explicit
// depth-first stack here, visiting the intervals in the recursion's order (same summation order as the oracle). ----
template <int P, int ORDER, class NODE>
__device__ __forceinline__ void integrate_gk_step(const NODE& node, double bl, double br, double* acc) {
    constexpr int NP = 2 * ORDER + 1;
    constexpr double X7[7] = {-0.960491268708020283423507092629080, -0.774596669241483377035853079956480, -0.405845151377397166906606412076961, 0.0,
                              0.405845151377397166906606412076961, 0.774596669241483377035853079956480, 0.960491268708020283423507092629080};
    constexpr double W7[7] = {0.104656226026467265193823857192073, 0.268488089868333440728569280666710, 0.401397414775962222905051818618432,
                              0.450916538658474142345110087045571, 0.401397414775962222905051818618432, 0.268488089868333440728569280666710,
                              0.104656226026467265193823857192073};
    constexpr double G3[3] = {0.555555555555555555555555555555556, 0.888888888888888888888888888888889, 0.555555555555555555555555555555556};
    constexpr double X3[3] = {-0.774596669241483377035853079956480, 0.0, 0.774596669241483377035853079956480};
    constexpr double G1[1] = {2.0};
    double sl[32], sr[32];
    int sd[32], sp = 1;
    sl[0] = bl; sr[0] = br; sd[0] = 0;
    while (sp > 0) {
        sp--;
        const double l = sl[sp], r = sr[sp];
        const int dep = sd[sp];
        double K[P], G[P], v[P];
#pragma unroll
        for (int q = 0; q < P; q++) { K[q] = 0.0; G[q] = 0.0; }
#pragma unroll
        for (int i = 0; i < NP; i++) {
            const double x = ORDER == 3 ? X7[i < 7 ? i : 0] : X3[i < 3 ? i : 0];
            const double w = ORDER == 3 ? W7[i < 7 ? i : 0] : G3[i < 3 ? i : 0];          // K3 weights = the 3-point Gauss weights
            node(0.5 * (r - l) * x + 0.5 * (l + r), v);
#pragma unroll
            for (int q = 0; q < P; q++) K[q] += w * v[q];
            if (i & 1) {
                const double g = ORDER == 3 ? G3[(i / 2) < 3 ? i / 2 : 0] : G1[0];
#pragma unroll
                for (int q = 0; q < P; q++) G[q] += g * v[q];
            }
        }
        double err = 0.0;
#pragma unroll
        for (int q = 0; q < P; q++) { K[q] *= 0.5 * (r - l); G[q] *= 0.5 * (r - l); err += fabs(K[q] - G[q]); }
        if (err < 1e-7 || dep >= 30) {
#pragma unroll
            for (int q = 0; q < P; q++) acc[q] += K[q];
        } else {
            const double mid = 0.5 * (l + r);
            sl[sp] = mid; sr[sp] = r; sd[sp] = dep + 1; sp++;      // right half waits
            sl[sp] = l; sr[sp] = mid; sd[sp] = dep + 1; sp++;      // left half next
        }
    }
}

// The member loop shared by the three quadrature kernels: a persistent grid of QUAD_WARPS-warp blocks, warp g takes
// members g, g + G, ... (static assignment => per-member results and the shared-p sum are reproducible), integrates the
// data intervals in the reference's order (src/quadrature_adjoint.jl:537-616) and hands the member's dp[P] to `sink`.
template <int P, class MAKE, class SINK>
__device__ __forceinline__ void quad_member_loop(int64_t N, int K, const double* saveat, double t0, double t1, double atol, double rtol,
                                                 double* qseg, double* qkey, int maxseg, double* l1_smem, const MAKE& make, const SINK& sink) {
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int64_t gw = (int64_t)blockIdx.x * QUAD_WARPS + wib, G = (int64_t)gridDim.x * QUAD_WARPS;
    // dynamic shared memory of the block: [QUAD_WARPS][QUAD_SKEYS] keys, then [QUAD_WARPS][quad_l1_blocks(maxseg)] block maxima
    const QuadScratch qs{qseg + (size_t)gw * maxseg * quad_segw<P>(), qkey + (size_t)gw * maxseg, l1_smem + (size_t)wib * QUAD_SKEYS,
                         l1_smem + (size_t)QUAD_WARPS * QUAD_SKEYS + (size_t)wib * quad_l1_blocks(maxseg), maxseg};
    for (int64_t i = gw; i < N; i += G) {
        double res[P], part[P];
#pragma unroll
        for (int q = 0; q < P; q++) res[q] = 0.0;
        auto ctx = make(i);
        bool ok = ctx.valid();
        if (ok && !ctx.empty()) {
            const QuadBracket root = ctx.root();
            auto add = [&](double lo, double hi) {
                ok = quadgk_warp<P>(ctx, root, lo, hi, atol, rtol, part, qs, lane) && ok;
#pragma unroll
                for (int q = 0; q < P; q++) res[q] += part[q];
            };
            if (K == 0) add(t0, t1);
            else {
                if (saveat[K - 1] != t1) add(saveat[K - 1], t1);
                for (int k = K - 2; k >= 0; k--) if (saveat[k] != saveat[k + 1]) add(saveat[k], saveat[k + 1]);
                if (saveat[0] != t0) add(t0, saveat[0]);
            }
        }
        if (!ok) {           // dense reverse solution overflowed, or out of segment capacity: fail loudly (NaN), never a silent partial
#pragma unroll
            for (int q = 0; q < P; q++) res[q] = __longlong_as_double(0x7ff8000000000000LL);
        }
        sink(i, res);
        __syncwarp();
    }
}

}  // namespace b200adj
