// quadgk_probe.cu -- one-warp probes of the warp-cooperative quadgk of QuadratureAdjoint (csrc/quadgk.cuh) and of the two
// production integrand contexts that feed it (ros23.cuh::RosQuadCtx, tsit5_adaptive.cuh::T5aQuadCtx), for
// tests/test_gpu_quadgk_probe.py.  The production device functions are called unchanged; this file only adds synthetic
// integrands, __global__ wrappers and extern "C" launchers over device pointers.  Test-only: it is not part of libb200adj.so.
//
// Every scratch buffer a probe hands to production code carries padding past what the production sizing asks for, and the
// dynamic shared allocation ends in a guard region filled with a sentinel, so that an out-of-range store is REPORTED (guard
// intact or not) instead of reaching memory the probe does not own.  Launchers wait for the kernel and return the
// cudaError_t (0 = success).
#include "handle.h"

using namespace b200adj;

namespace {

constexpr int GUARD = 64;                 // doubles of sentinel after the shared layout
constexpr int PAD = 64;                   // extra segment records / keys after the production-sized global scratch
constexpr long long SENTINEL = 0x5a5a5a5a5a5a5a5aLL;
constexpr long long POISON = 0x7ff4000000000badLL;     // a NaN: scratch the production code reads before writing would show

__device__ bool guard_intact(const double* g) {
    bool ok = true;
    for (int i = threadIdx.x & 31; i < GUARD; i += 32) ok = ok && __double_as_longlong(g[i]) == SENTINEL;
    return __all_sync(0xffffffffu, ok);
}
__device__ void fill_smem(double* s, int n_poison, int n_total) {
    for (int i = threadIdx.x; i < n_total; i += blockDim.x) s[i] = __longlong_as_double(i < n_poison ? POISON : SENTINEL);
}

// ---- synthetic integrands: f_q(t), q < P ----
//   kind 0: polynomial   sum_k c[q (deg + 1) + k] t^k (Horner)
//   kind 1: step         sum_j s[j P + q] [t >= jt[j]]
//   kind 2: polynomial, NaN where |t - tnan| < 1e-12 (one node of the root segment)
struct Synth {
    int kind, deg; const double* c; int nj; const double* jt; const double* js; double tnan, scale;
    int* calls;                            // lane 0 counts gk15_pair calls (= segments of the run: 1 + bisections)
};
template <int P>
__device__ __forceinline__ void synth_eval(const Synth& s, double t, int lane, double* out) {
    if (lane == 0) (*s.calls)++;
#pragma unroll
    for (int q = 0; q < P; q++) out[q] = 0.0;
    if (s.kind == 1) {
        for (int j = 0; j < s.nj; j++)
            if (t >= s.jt[j]) {
#pragma unroll
                for (int q = 0; q < P; q++) out[q] += s.js[j * P + q];
            }
    } else {
#pragma unroll
        for (int q = 0; q < P; q++) {
            double v = s.c[q * (s.deg + 1) + s.deg];
            for (int k = s.deg - 1; k >= 0; k--) v = v * t + s.c[q * (s.deg + 1) + k];
            out[q] = v;
        }
        if (s.kind == 2 && fabs(t - s.tnan) < 1e-12) {
#pragma unroll
            for (int q = 0; q < P; q++) out[q] = __longlong_as_double(0x7ff8000000000000LL);
        }
    }
#pragma unroll
    for (int q = 0; q < P; q++) out[q] *= s.scale;
}
template <int P>
struct SynthF {
    Synth s;
    __device__ __forceinline__ bool valid() const { return true; }
    __device__ __forceinline__ bool empty() const { return false; }
    __device__ __forceinline__ QuadBracket root() const { return QuadBracket{0, 0, 0, 0}; }
    __device__ __forceinline__ void eval(double t, const QuadBracket&, int lane, double* out, int* fiv, int* riv) const {
        *fiv = 0; *riv = 0;
        synth_eval<P>(s, t, lane, out);
    }
};

// ---- probe_coop_count: one warp, every lane its own t ----
__global__ void coop_count_kernel(int asc, const double* knots, int first, int cnt, const double* t, int* out) {
    const int lane = threadIdx.x;
    auto knot = [&](int j) { return __ldg(knots + j); };
    out[lane] = asc ? coop_count<true>(knot, first, cnt, t[lane], lane) : coop_count<false>(knot, first, cnt, t[lane], lane);
}

__global__ void warp_argmax_kernel(const double* v, const int* present, int* out) {
    out[threadIdx.x] = warp_argmax_lane(v[threadIdx.x], present[threadIdx.x] != 0);
}

// ---- the queue arg-max on crafted keys: skey[QUAD_SKEYS] and l1[nb] copied into the production shared layout (keys, then
// block maxima, then the guard), key = the global key array ----
__global__ void queue_argmax_kernel(const double* skey, const double* key, const double* l1, int nseg, int* w_out, double* ew_out, int* guard_ok) {
    extern __shared__ double sm[];
    const int nb = (nseg + 31) >> 5, lane = threadIdx.x;
    fill_smem(sm, QUAD_SKEYS + nb, QUAD_SKEYS + nb + GUARD);
    __syncwarp();
    for (int i = lane; i < QUAD_SKEYS; i += 32) sm[i] = skey[i];
    for (int i = lane; i < nb; i += 32) sm[QUAD_SKEYS + i] = l1[i];
    __syncwarp();
    const QuadScratch q{nullptr, const_cast<double*>(key), sm, sm + QUAD_SKEYS, nseg};
    const QuadPick pk = quad_queue_argmax(q, nseg, lane);
    const bool g = guard_intact(sm + QUAD_SKEYS + nb);
    if (lane == 0) { w_out[0] = pk.w; w_out[1] = pk.bi; ew_out[0] = pk.ew; guard_ok[0] = g; }
}

// ---- quadgk_warp on a synthetic integrand, one warp; shared layout of one warp of quad_member_loop + guard ----
template <int P>
__global__ void quadgk_kernel(Synth s, double a, double b, double atol, double rtol, int maxseg, double* seg, double* key,
                              double* out, int* info, double* ab) {
    extern __shared__ double sm[];
    const int lane = threadIdx.x, nl1 = quad_l1_blocks(maxseg);
    fill_smem(sm, QUAD_SKEYS + nl1, QUAD_SKEYS + nl1 + GUARD);
    if (lane == 0) *s.calls = 0;
    __syncwarp();
    const QuadScratch q{seg, key, sm, sm + QUAD_SKEYS, maxseg};
    double res[P];
    const bool ok = quadgk_warp<P>(SynthF<P>{s}, QuadBracket{0, 0, 0, 0}, a, b, atol, rtol, res, q, lane);
    __syncwarp();
    const int n = *s.calls;
    const bool g = guard_intact(sm + QUAD_SKEYS + nl1);
    constexpr int SEGW = quad_segw<P>();
    for (int i = lane; i < n && i < maxseg + PAD; i += 32) { ab[2 * i] = seg[(size_t)i * SEGW]; ab[2 * i + 1] = seg[(size_t)i * SEGW + 1]; }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < P; k++) out[k] = res[k];
        info[0] = ok; info[1] = n; info[2] = g;
    }
}

// ---- quad_member_loop with a persistent grid of `grid` blocks of QUAD_WARPS warps.  Member i integrates the step function
// jt[joff[i] ..], js[(joff[i] + j) P + q] (nj[i] jumps) times mult[i]; dp[q N + i] = its result, calls[i] = its gk15_pair
// calls over all data intervals.  Dynamic shared memory: quad_smem(maxseg) + guard, guard_ok[block].  K = 0 (one data interval
// per member): l1_bad counts the blocks whose maximum, in the table where quad_smem places this warp's (stride
// quad_l1_blocks(maxseg)), is not bit for bit the maximum of the keys the warp's last member left behind. ----
constexpr int ML_P = 3;
__global__ void __launch_bounds__(QUAD_WARPS * 32) member_loop_kernel(int64_t N, int K, const double* saveat, double t0, double t1, double atol,
                                                                    double rtol, double* qseg, double* qkey, int maxseg, const int* joff,
                                                                    const int* nj, const double* mult, const double* jt, const double* js,
                                                                    int* calls, double* dp, int nsm, int* guard_ok, unsigned* l1_bad) {
    extern __shared__ double sm[];                  // nsm = quad_smem(maxseg) / 8 doubles, then the guard
    fill_smem(sm, nsm, nsm + GUARD);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    auto make = [&](int64_t i) {
        return SynthF<ML_P>{Synth{1, 0, nullptr, nj[i], jt + joff[i], js + (size_t)joff[i] * ML_P, 0.0, mult[i], calls + i}};
    };
    auto sink = [&](int64_t i, const double* res) {
        if (lane == 0) {
#pragma unroll
            for (int q = 0; q < ML_P; q++) dp[(int64_t)q * N + i] = res[q];
        }
    };
    quad_member_loop<ML_P>(N, K, saveat, t0, t1, atol, rtol, qseg, qkey, maxseg, sm, make, sink);
    __syncthreads();
    bool g = true;
    for (int i = threadIdx.x; i < GUARD; i += blockDim.x) g = g && __double_as_longlong(sm[nsm + i]) == SENTINEL;
    g = __syncthreads_and(g);
    if (threadIdx.x == 0) guard_ok[blockIdx.x] = g;
    const int wib = threadIdx.x >> 5;
    const int64_t gw = (int64_t)blockIdx.x * QUAD_WARPS + wib, G = (int64_t)gridDim.x * QUAD_WARPS;
    if (K == 0 && gw < N) {
        const int n = calls[gw + G * ((N - 1 - gw) / G)];
        const double* skey = sm + (size_t)wib * QUAD_SKEYS;
        const double* key = qkey + (size_t)gw * maxseg;
        const double* l1 = sm + (size_t)QUAD_WARPS * QUAD_SKEYS + (size_t)wib * quad_l1_blocks(maxseg);
        unsigned bad = 0;
        for (int b = 0; b < ((n + 31) >> 5); b++) {
            const int k = b * 32 + lane;
            const double m = warp_max(k < n ? (k < QUAD_SKEYS ? skey[k] : key[k]) : 0.0);
            bad += __double_as_longlong(m) != __double_as_longlong(l1[b]) ? 1u : 0u;
        }
        if (lane == 0 && bad) atomicAdd(l1_bad, bad);
    }
}

// ---- the production integrand contexts on synthetic member-major records.  ProbeFam::vjp_p is the bilinear form
// out[q] = sum_jk B[q][j][k] y[j] lam[k]; the checking wrapper recomputes the forward interval and the reverse record of every
// lookup by a scan over ALL knots and counts bad[0] = mismatches, bad[1] = expected index outside the segment's bracket. ----
constexpr int CD = 2, CP = 3;
__constant__ double PROBE_B[CP][CD][CD];
struct ProbeFam {
    static constexpr int D = CD, P = CP;
    static __device__ __forceinline__ void vjp_p(const double* y, const double*, const double* lam, double* out) {
#pragma unroll
        for (int q = 0; q < P; q++) {
            double s = 0.0;
#pragma unroll
            for (int j = 0; j < D; j++)
#pragma unroll
                for (int k = 0; k < D; k++) s += PROBE_B[q][j][k] * y[j] * lam[k];
            out[q] = s;
        }
    }
};
template <class Ctx>
struct Checked {
    Ctx c; const double* ftT; const double* rend; int nf, nrev; unsigned* bad; int* calls;
    __device__ __forceinline__ void eval(double t, const QuadBracket& br, int lane, double* out, int* fiv, int* riv) const {
        c.eval(t, br, lane, out, fiv, riv);
        if (lane == 0) (*calls)++;
        int iv = 0, lo = 0;
        for (int j = 1; j < nf; j++) iv += __ldg(ftT + j) < t ? 1 : 0;         // interior forward knots < t (left-continuous)
        for (int j = 0; j < nrev - 1; j++) lo += __ldg(rend + j) > t ? 1 : 0;  // reverse ends > t (ends descend)
        if (iv != *fiv || lo != *riv) atomicAdd(bad, 1u);
        if (iv < br.flo || iv > br.fhi || lo < br.rlo || lo > br.rhi) atomicAdd(bad + 1, 1u);
    }
};
template <class Ctx>
__device__ void ctx_run(const Ctx& ctx, const double* ftT, const double* rend, int nf, int nrev, double a, double b, double atol,
                        double rtol, int maxseg, double* seg, double* key, double* out, int* info, unsigned* bad) {
    extern __shared__ double sm[];
    const int lane = threadIdx.x, nl1 = quad_l1_blocks(maxseg);
    fill_smem(sm, QUAD_SKEYS + nl1, QUAD_SKEYS + nl1 + GUARD);
    if (lane == 0) { info[1] = 0; bad[0] = 0; bad[1] = 0; }
    __syncwarp();
    const QuadScratch q{seg, key, sm, sm + QUAD_SKEYS, maxseg};
    const Checked<Ctx> f{ctx, ftT, rend, nf, nrev, bad, info + 1};
    double res[CP];
    const bool ok = quadgk_warp<CP>(f, ctx.root(), a, b, atol, rtol, res, q, lane);
    __syncwarp();
    const bool g = guard_intact(sm + QUAD_SKEYS + nl1);
    if (lane == 0) {
        for (int k = 0; k < CP; k++) out[k] = res[k];
        info[0] = ok; info[2] = g;
    }
}
__global__ void ros_ctx_kernel(const double* ftT, const double* frecT, const double* rrec, const double* rend, int nf, int nrev, double a, double b,
                               double atol, double rtol, int maxseg, double* seg, double* key, double* out, int* info, unsigned* bad) {
    const RosQuadCtx<ProbeFam, CD, CP> c{ftT, frecT, rrec, rend, nf, nrev, {0.0, 0.0, 0.0}};
    ctx_run(c, ftT, rend, nf, nrev, a, b, atol, rtol, maxseg, seg, key, out, info, bad);
}
__global__ void t5a_ctx_kernel(const __grid_constant__ T5aArgs args, const double* ftT, const double* frecT, const double* rrec, const double* rend,
                               int nf, int nrev, double a, double b, double atol, double rtol, int maxseg, double* seg, double* key, double* out,
                               int* info, unsigned* bad) {
    const T5aQuadCtx<ProbeFam, CD, CP> c{args, ftT, frecT, rrec, rend, nf, nrev, {0.0, 0.0, 0.0}};
    ctx_run(c, ftT, rend, nf, nrev, a, b, atol, rtol, maxseg, seg, key, out, info, bad);
}

int finish() {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    return (int)cudaDeviceSynchronize();
}
size_t warp_smem(int maxseg) { return (size_t)(QUAD_SKEYS + quad_l1_blocks(maxseg) + GUARD) * sizeof(double); }
// padded, poisoned global segment scratch of one warp
struct Scratch {
    double* seg = nullptr; double* key = nullptr;
    int alloc(size_t records, int segw) {
        if (cudaMalloc(&seg, (records + PAD) * segw * sizeof(double)) != cudaSuccess) return 1;
        if (cudaMalloc(&key, (records + PAD) * sizeof(double)) != cudaSuccess) return 1;
        cudaMemset(seg, 0xff, (records + PAD) * segw * sizeof(double));      // all-ones bits: a NaN
        cudaMemset(key, 0xff, (records + PAD) * sizeof(double));
        return 0;
    }
    ~Scratch() { cudaFree(seg); cudaFree(key); }
};
int set_smem(const void* kernel, size_t bytes) {
    return bytes > 48 * 1024 ? (int)cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) : 0;
}

template <int P>
int run_quadgk(const Synth& s, double a, double b, double atol, double rtol, int maxseg, double* out, int* info, double* ab) {
    Scratch sc;
    if (sc.alloc(maxseg, quad_segw<P>())) return (int)cudaErrorMemoryAllocation;
    const size_t sm = warp_smem(maxseg);
    if (int e = set_smem((const void*)quadgk_kernel<P>, sm)) return e;
    quadgk_kernel<P><<<1, 32, sm>>>(s, a, b, atol, rtol, maxseg, sc.seg, sc.key, out, info, ab);
    return finish();
}

}  // namespace

extern "C" {

// the production layout of the quadrature kernels: dynamic shared bytes per block, block maxima per warp
void probe_layout(int maxseg, long long* smem_bytes, int* l1_per_warp, int* warps, int* skeys) {
    *smem_bytes = (long long)quad_smem(maxseg);
    *l1_per_warp = quad_l1_blocks(maxseg);
    *warps = QUAD_WARPS;
    *skeys = QUAD_SKEYS;
}

int probe_coop_count(int asc, const double* knots, int first, int cnt, const double* t, int* out) {
    coop_count_kernel<<<1, 32>>>(asc, knots, first, cnt, t, out);
    return finish();
}

int probe_warp_argmax(const double* v, const int* present, int* out) {
    warp_argmax_kernel<<<1, 32>>>(v, present, out);
    return finish();
}

// w_out[2] = (winning segment, winning block), ew_out[1] = its key
int probe_queue_argmax(const double* skey, const double* key, const double* l1, int nseg, int* w_out, double* ew_out, int* guard_ok) {
    const size_t sm = (size_t)(QUAD_SKEYS + ((nseg + 31) >> 5) + GUARD) * sizeof(double);
    if (int e = set_smem((const void*)queue_argmax_kernel, sm)) return e;
    queue_argmax_kernel<<<1, 32, sm>>>(skey, key, l1, nseg, w_out, ew_out, guard_ok);
    return finish();
}

// info[3] = (ok, segments, guard intact); ab[(maxseg + 64)][2] = final (a, b) of every segment; calls: one device int
int probe_quadgk(int kind, int P, double a, double b, double atol, double rtol, int maxseg, int deg, const double* coef, int nj,
                 const double* jt, const double* js, double tnan, int* calls, double* out, int* info, double* ab) {
    const Synth s{kind, deg, coef, nj, jt, js, tnan, 1.0, calls};
    switch (P) {
        case 1: return run_quadgk<1>(s, a, b, atol, rtol, maxseg, out, info, ab);
        case 3: return run_quadgk<3>(s, a, b, atol, rtol, maxseg, out, info, ab);
        case 4: return run_quadgk<4>(s, a, b, atol, rtol, maxseg, out, info, ab);
        case 8: return run_quadgk<8>(s, a, b, atol, rtol, maxseg, out, info, ab);
        default: return (int)cudaErrorInvalidValue;
    }
}

int probe_member_loop(int grid, long long N, int K, const double* saveat, double t0, double t1, double atol, double rtol, int maxseg,
                      const int* joff, const int* nj, const double* mult, const double* jt, const double* js, int* calls, double* dp,
                      int* guard_ok, unsigned* l1_bad) {
    Scratch sc;
    if (sc.alloc((size_t)grid * QUAD_WARPS * maxseg, quad_segw<ML_P>())) return (int)cudaErrorMemoryAllocation;
    const size_t sm = quad_smem(maxseg) + GUARD * sizeof(double);
    if (int e = set_smem((const void*)member_loop_kernel, sm)) return e;
    member_loop_kernel<<<grid, QUAD_WARPS * 32, sm>>>(N, K, saveat, t0, t1, atol, rtol, sc.seg, sc.key, maxseg, joff, nj, mult, jt, js, calls, dp,
                                                      (int)(quad_smem(maxseg) / sizeof(double)), guard_ok, l1_bad);
    return finish();
}

// kind 0: Rosenbrock23 records (RosQuadCtx), 1: adaptive Tsit5 records (T5aQuadCtx; R[7][4] = the dense-output polynomials).
// B[P][D][D] (host) = the bilinear form.  info[3] = (ok, segments, guard intact), bad[2] = (mismatches, outside the bracket).
int probe_ctx(int kind, const double* B, const double* R, const double* ftT, const double* frecT, const double* rrec, const double* rend,
              int nf, int nrev, double a, double b, double atol, double rtol, int maxseg, double* out, int* info, unsigned* bad) {
    if (cudaMemcpyToSymbol(PROBE_B, B, sizeof(double) * CP * CD * CD) != cudaSuccess) return (int)cudaGetLastError();
    Scratch sc;
    if (sc.alloc(maxseg, quad_segw<CP>())) return (int)cudaErrorMemoryAllocation;
    const size_t sm = warp_smem(maxseg);
    if (kind == 0) {
        if (int e = set_smem((const void*)ros_ctx_kernel, sm)) return e;
        ros_ctx_kernel<<<1, 32, sm>>>(ftT, frecT, rrec, rend, nf, nrev, a, b, atol, rtol, maxseg, sc.seg, sc.key, out, info, bad);
    } else {
        T5aArgs args;
        memset(&args, 0, sizeof(args));
        memcpy(args.R, R, sizeof(args.R));
        if (int e = set_smem((const void*)t5a_ctx_kernel, sm)) return e;
        t5a_ctx_kernel<<<1, 32, sm>>>(args, ftT, frecT, rrec, rend, nf, nrev, a, b, atol, rtol, maxseg, sc.seg, sc.key, out, info, bad);
    }
    return finish();
}

}  // extern "C"
