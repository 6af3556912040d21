// disp_mlp.cu -- launchers of the MLP-family kernels: CUDA-core fp64 / fp32 (mlp.cuh) and the wgmma bf16 path (mlp_tc.cuh)
#include "handle.h"
namespace b200adj {
namespace {
template <class T>
int mlp_forward_launch(Handle* h, const void* u0, const void* p, void* saved, int32_t* status) {
    MlpArgs<T> a;
    memset(&a, 0, sizeof(a));
    a.u0 = (const T*)u0; a.p = (const T*)p; a.ckpt = (T*)h->d_ckpt; a.saved = (T*)saved; a.save_of_step = h->d_fwd_save_of_step;
    a.status = status; a.N = h->cfg.N; a.S = h->S; a.tb = h->tb;
    if (h->nev > 0) { a.event_of_step = h->d_event_of_step; a.ev_s = h->d_ev_s; a.ev_c = h->d_ev_c; }
    const size_t smem = sizeof(MlpSmem<T>);
    if (cudaFuncSetAttribute(mlp_forward_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return B200ADJ_ERR_CUDA;
    mlp_forward_kernel<T><<<h->grid, MLP_THREADS, smem, h->stream>>>(a);
    h->launches++;
    return 0;
}
// BF16_F32ACC: two layouts of the same tensor-core kernels.  32 members per CTA (mlp_tc.cuh: 4x more CTAs, a quarter of the
// per-thread work per stage) while its CTAs fit in one wave of 2 per SM; 128 members per CTA (mlp_tc_wide.cuh: highest
// throughput) beyond that.
static bool mlp_tc_narrow(const Handle* h) { return (h->cfg.N + TC_MEM - 1) / TC_MEM <= 2 * (int64_t)h->nsm; }
int mlp_tc_forward_launch(Handle* h, const void* u0, const void* p, void* saved, int32_t* status) {
    MlpArgs<float> a;
    memset(&a, 0, sizeof(a));
    a.u0 = (const float*)u0; a.p = (const float*)p; a.ckpt = (float*)h->d_ckpt; a.saved = (float*)saved; a.save_of_step = h->d_fwd_save_of_step;
    a.status = status; a.N = h->cfg.N; a.S = h->S; a.tb = h->tb; a.kst = h->d_kst;
    if (mlp_tc_narrow(h)) {
        const size_t smem = sizeof(TcSmem) + 128;
        if (cudaFuncSetAttribute(mlp_tc_forward_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return B200ADJ_ERR_CUDA;
        mlp_tc_forward_kernel<0><<<(int)((h->cfg.N + TC_MEM - 1) / TC_MEM), TC_M, smem, h->stream>>>(a);
    } else {
        const size_t smem = sizeof(TcwSmem) + 128;
        if (cudaFuncSetAttribute(mlp_tcw_forward_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return B200ADJ_ERR_CUDA;
        mlp_tcw_forward_kernel<0><<<(int)((h->cfg.N + TCW_M - 1) / TCW_M), TCW_M, smem, h->stream>>>(a);
    }
    h->launches++;
    return 0;
}
int mlp_tc_reverse_launch(Handle* h, const void* dLdu, void* du0, void* dp) {
    const b200adj_cfg& c = h->cfg;
    MlpArgs<float> a;
    memset(&a, 0, sizeof(a));
    a.p = (const float*)h->cur_p; a.ckpt = (float*)h->d_ckpt; a.save_of_step = h->d_save_of_step; a.dLdu = (const float*)dLdu;
    a.du0 = (float*)du0; a.partials = (float*)h->d_partials; a.dp = (float*)dp; a.N = c.N; a.S = h->S; a.tb = h->tb; a.kst = h->d_kst;
    for (int j = 0; j < 4; j++) { a.cost_a[j] = h->cost_av[j]; a.cost_b[j] = h->cost_bv[j]; } a.flags = kernel_flags(h) & KF_NO_START;
    const bool narrow = mlp_tc_narrow(h), ex = c.cost_kind == B200ADJ_COST_EXPLICIT;
    const size_t smem = (narrow ? sizeof(TcSmem) : sizeof(TcwSmem)) + 128;
    const int grid = narrow ? (int)((c.N + TC_MEM - 1) / TC_MEM) : (int)((c.N + TCW_M - 1) / TCW_M);
#define B200_TC_REV(KERNEL, THREADS)                                                                                         \
    do {                                                                                                                     \
        if (cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return B200ADJ_ERR_CUDA; \
        KERNEL<<<grid, THREADS, smem, h->stream>>>(a);                                                                       \
    } while (0)
#define B200_TC_REV2(COSTV, GAUSSV)                                                                                      \
    do { if (narrow) B200_TC_REV((mlp_tc_reverse_kernel<COSTV, GAUSSV>), TC_M); else B200_TC_REV((mlp_tcw_reverse_kernel<COSTV, GAUSSV>), TCW_M); } while (0)
    const bool gauss = c.sensealg == B200ADJ_SA_GAUSS;
    if (gauss) { if (ex) B200_TC_REV2(COST_EXPLICIT, true); else B200_TC_REV2(COST_AFFINE, true); }
    else { if (ex) B200_TC_REV2(COST_EXPLICIT, false); else B200_TC_REV2(COST_AFFINE, false); }
#undef B200_TC_REV2
#undef B200_TC_REV
    mlp_reduce_kernel<float><<<(MLP_P + 255) / 256, 256, 0, h->stream>>>((const float*)h->d_partials, (float*)dp, grid);
    h->launches += 2;
    return 0;
}
template <class T>
int mlp_reverse_launch(Handle* h, const void* dLdu, void* du0, void* dp) {
    const b200adj_cfg& c = h->cfg;
    MlpArgs<T> a;
    memset(&a, 0, sizeof(a));
    a.p = (const T*)h->cur_p; a.ckpt = (T*)h->d_ckpt; a.save_of_step = h->d_save_of_step; a.dLdu = (const T*)dLdu;
    a.du0 = (T*)du0; a.partials = (T*)h->d_partials; a.dp = (T*)dp; a.N = c.N; a.S = h->S; a.tb = h->tb;
    for (int j = 0; j < 4; j++) { a.cost_a[j] = h->cost_av[j]; a.cost_b[j] = h->cost_bv[j]; } a.flags = kernel_flags(h) & KF_NO_START;
    const size_t smem = sizeof(MlpSmem<T>);
    if (h->nev > 0) { a.event_of_step = h->d_event_of_step; a.ev_s = h->d_ev_s; a.ev_c = h->d_ev_c; }
#define B200_MLP_REV(COSTV, GAUSSV)                                                                                         \
    do {                                                                                                                    \
        if (cudaFuncSetAttribute(mlp_reverse_kernel<T, COSTV, GAUSSV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return B200ADJ_ERR_CUDA; \
        mlp_reverse_kernel<T, COSTV, GAUSSV><<<h->grid, MLP_THREADS, smem, h->stream>>>(a);                                 \
    } while (0)
    const bool ex = c.cost_kind == B200ADJ_COST_EXPLICIT;
    if (c.sensealg == B200ADJ_SA_GAUSS) { if (ex) B200_MLP_REV(COST_EXPLICIT, true); else B200_MLP_REV(COST_AFFINE, true); }
    else { if (ex) B200_MLP_REV(COST_EXPLICIT, false); else B200_MLP_REV(COST_AFFINE, false); }
#undef B200_MLP_REV
    mlp_reduce_kernel<T><<<(MLP_P + 255) / 256, 256, 0, h->stream>>>((const T*)h->d_partials, (T*)dp, h->grid);
    h->launches += 2;
    return 0;
}
}  // namespace

int mlp_forward_dispatch(Handle* h, const void* u0, const void* p, void* saved, int32_t* status) {
    const b200adj_cfg& c = h->cfg;
    return is_mlp_tc(h) ? mlp_tc_forward_launch(h, u0, p, saved, status)
         : c.dtype != B200ADJ_F64 ? mlp_forward_launch<float>(h, u0, p, saved, status) : mlp_forward_launch<double>(h, u0, p, saved, status);
}
int mlp_reverse_dispatch(Handle* h, const void* dLdu, void* du0, void* dp) {
    const b200adj_cfg& c = h->cfg;
    return is_mlp_tc(h) ? mlp_tc_reverse_launch(h, dLdu, du0, dp)
         : c.dtype != B200ADJ_F64 ? mlp_reverse_launch<float>(h, dLdu, du0, dp) : mlp_reverse_launch<double>(h, dLdu, du0, dp);
}
}  // namespace b200adj
