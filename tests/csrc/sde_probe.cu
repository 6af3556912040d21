// sde_probe.cu -- the random-number pieces of the SDE kernels (csrc/sde_em.cuh) evaluated on caller-supplied inputs, for
// tests/test_gpu_sde_probe.py: b200adj::philox4x32_10 beside the toolkit's own curand_Philox4x32_10 on the same words,
// b200adj::normal_pair, and b200adj::wiener_increment<M> for M = 1, 2, 3 (the odd M pins the layout of a last, unpaired
// component, which no built-in family reaches).  One kernel of its own; no library kernel is launched.  Test-only: it is
// not part of libb200adj.so.  The entry point copies in, launches, copies out and returns the cudaError_t (0 = success).
#include <curand_philox4x32_x.h>
#include "sde_em.cuh"

using namespace b200adj;

namespace {

struct ProbeArgs {
    int n; const uint32_t* ctr; const uint32_t* key; uint32_t* ours; uint32_t* theirs;
    int nz; const uint64_t* seed; const uint64_t* member; const uint32_t* step; const uint32_t* pair; const double* sqrth;
    double* z; double* w;
};

__global__ void sde_probe_kernel(ProbeArgs a) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.n) {
        const uint32_t* c = a.ctr + 4 * t;
        const uint32_t* k = a.key + 2 * t;
        philox4x32_10(c[0], c[1], c[2], c[3], k[0], k[1], a.ours + 4 * t);
        const uint4 r = curand_Philox4x32_10(make_uint4(c[0], c[1], c[2], c[3]), make_uint2(k[0], k[1]));
        a.theirs[4 * t] = r.x; a.theirs[4 * t + 1] = r.y; a.theirs[4 * t + 2] = r.z; a.theirs[4 * t + 3] = r.w;
    }
    if (t < a.nz) {
        normal_pair(a.seed[t], a.member[t], a.step[t], a.pair[t], a.z + 2 * t, a.z + 2 * t + 1);
        double* w = a.w + 6 * t;
        wiener_increment<1>(a.seed[t], a.member[t], a.step[t], a.sqrth[t], w);
        wiener_increment<2>(a.seed[t], a.member[t], a.step[t], a.sqrth[t], w + 1);
        wiener_increment<3>(a.seed[t], a.member[t], a.step[t], a.sqrth[t], w + 3);
    }
}

template <class T>
cudaError_t to_device(T** d, const T* h, size_t count) {
    cudaError_t r = cudaMalloc(d, (count ? count : 1) * sizeof(T));
    if (r == cudaSuccess && h && count) r = cudaMemcpy(*d, h, count * sizeof(T), cudaMemcpyHostToDevice);
    return r;
}

}  // namespace

extern "C" {

// n Philox cases: ctr[n][4], key[n][2] -> ours[n][4] (b200adj::philox4x32_10), theirs[n][4] (curand_Philox4x32_10).
// nz generator cases: seed[nz], member[nz], step[nz], pair[nz], sqrth[nz] -> z[nz][2] = normal_pair(seed, member, step,
// pair) and w[nz][6] = wiener_increment<1> (1 value), <2> (2 values), <3> (3 values) of (seed, member, step, sqrth).
int probe_sde_random(int n, const uint32_t* ctr, const uint32_t* key, uint32_t* ours, uint32_t* theirs,
                     int nz, const uint64_t* seed, const uint64_t* member, const uint32_t* step, const uint32_t* pair,
                     const double* sqrth, double* z, double* w) {
    ProbeArgs a;
    a.n = n; a.nz = nz;
    uint32_t *dc = nullptr, *dk = nullptr, *dours = nullptr, *dtheirs = nullptr, *dstep = nullptr, *dpair = nullptr;
    uint64_t *dseed = nullptr, *dmember = nullptr;
    double *dsq = nullptr, *dz = nullptr, *dw = nullptr;
    cudaError_t r = to_device(&dc, ctr, 4 * (size_t)n);
    if (r == cudaSuccess) r = to_device(&dk, key, 2 * (size_t)n);
    if (r == cudaSuccess) r = to_device<uint32_t>(&dours, nullptr, 4 * (size_t)n);
    if (r == cudaSuccess) r = to_device<uint32_t>(&dtheirs, nullptr, 4 * (size_t)n);
    if (r == cudaSuccess) r = to_device(&dseed, seed, (size_t)nz);
    if (r == cudaSuccess) r = to_device(&dmember, member, (size_t)nz);
    if (r == cudaSuccess) r = to_device(&dstep, step, (size_t)nz);
    if (r == cudaSuccess) r = to_device(&dpair, pair, (size_t)nz);
    if (r == cudaSuccess) r = to_device(&dsq, sqrth, (size_t)nz);
    if (r == cudaSuccess) r = to_device<double>(&dz, nullptr, 2 * (size_t)nz);
    if (r == cudaSuccess) r = to_device<double>(&dw, nullptr, 6 * (size_t)nz);
    if (r == cudaSuccess) {
        a.ctr = dc; a.key = dk; a.ours = dours; a.theirs = dtheirs;
        a.seed = dseed; a.member = dmember; a.step = dstep; a.pair = dpair; a.sqrth = dsq; a.z = dz; a.w = dw;
        const int work = n > nz ? n : nz;
        if (work > 0) sde_probe_kernel<<<(work + 127) / 128, 128>>>(a);
        r = cudaGetLastError();
    }
    if (r == cudaSuccess) r = cudaDeviceSynchronize();
    if (r == cudaSuccess && n) r = cudaMemcpy(ours, dours, 4 * (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost);
    if (r == cudaSuccess && n) r = cudaMemcpy(theirs, dtheirs, 4 * (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost);
    if (r == cudaSuccess && nz) r = cudaMemcpy(z, dz, 2 * (size_t)nz * sizeof(double), cudaMemcpyDeviceToHost);
    if (r == cudaSuccess && nz) r = cudaMemcpy(w, dw, 6 * (size_t)nz * sizeof(double), cudaMemcpyDeviceToHost);
    cudaFree(dc); cudaFree(dk); cudaFree(dours); cudaFree(dtheirs); cudaFree(dseed); cudaFree(dmember);
    cudaFree(dstep); cudaFree(dpair); cudaFree(dsq); cudaFree(dz); cudaFree(dw);
    return (int)r;
}

}  // extern "C"
