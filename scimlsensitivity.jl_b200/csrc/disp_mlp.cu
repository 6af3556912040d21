// disp_mlp.cu -- launchers of the MLP-family kernels: CUDA-core fp64 / fp32 (mlp.cuh) and the wgmma bf16 path (mlp_tc.cuh)
#include "handle.h"
namespace b200adj {
namespace {
// the arguments every MLP kernel reads (the preset-time events only where the handle has them: CUDA-core kernels)
template <class T>
MlpArgs<T> mlp_args(const Handle* h) {
    MlpArgs<T> a;
    memset(&a, 0, sizeof(a));
    a.ckpt = (T*)h->d_ckpt; a.N = h->cfg.N; a.S = h->S; a.tb = h->tb; a.kst = h->d_kst;
    if (h->nev > 0) { a.event_of_step = h->d_event_of_step; a.ev_s = h->d_ev_s; a.ev_c = h->d_ev_c; }
    return a;
}
template <class T>
MlpArgs<T> mlp_fwd_args(const Handle* h, const void* u0, const void* p, void* saved, int32_t* status) {
    MlpArgs<T> a = mlp_args<T>(h);
    a.u0 = (const T*)u0; a.p = (const T*)p; a.saved = (T*)saved; a.save_of_step = h->d_fwd_save_of_step; a.status = status;
    return a;
}
template <class T>
MlpArgs<T> mlp_rev_args(const Handle* h, const void* dLdu, void* du0, void* dp) {
    MlpArgs<T> a = mlp_args<T>(h);
    a.p = (const T*)h->cur_p; a.save_of_step = h->d_save_of_step; a.dLdu = (const T*)dLdu;
    a.du0 = (T*)du0; a.partials = (T*)h->d_partials; a.dp = (T*)dp;
    for (int j = 0; j < 4; j++) { a.cost_a[j] = h->cost_av[j]; a.cost_b[j] = h->cost_bv[j]; }
    a.flags = kernel_flags(h) & KF_NO_START;
    return a;
}
// the reverse kernel's per-block dp partials summed into dp
template <class T>
int mlp_reduce(Handle* h, void* dp, int nblocks) {
    return launch_kernel(h, mlp_reduce_kernel<T>, (MLP_P + 255) / 256, 256, 0, (const T*)h->d_partials, (T*)dp, nblocks);
}
// BF16_F32ACC: two layouts of the same tensor-core kernels.  32 members per CTA (mlp_tc.cuh: 4x more CTAs, a quarter of the
// per-thread work per stage) while its CTAs fit in one wave of 2 per SM; 128 members per CTA (mlp_tc_wide.cuh: highest
// throughput) beyond that.  Returns the grid in `grid`.
int mlp_tc_launch(Handle* h, void (*narrow)(MlpArgs<float>), void (*wide)(MlpArgs<float>), const MlpArgs<float>& a, int& grid) {
    if ((h->cfg.N + TC_MEM - 1) / TC_MEM <= 2 * (int64_t)h->nsm) {
        grid = (int)((h->cfg.N + TC_MEM - 1) / TC_MEM);
        return launch_kernel(h, narrow, grid, TC_M, sizeof(TcSmem) + 128, a);
    }
    grid = (int)((h->cfg.N + TCW_M - 1) / TCW_M);
    return launch_kernel(h, wide, grid, TCW_M, sizeof(TcwSmem) + 128, a);
}
}  // namespace

int mlp_forward_dispatch(Handle* h, const void* u0, const void* p, void* saved, int32_t* status) {
    if (is_mlp_tc(h)) {
        int grid;
        return mlp_tc_launch(h, mlp_tc_forward_kernel<0>, mlp_tcw_forward_kernel<0>, mlp_fwd_args<float>(h, u0, p, saved, status), grid);
    }
    auto go = [&](auto t) {
        using T = decltype(t);
        return launch_kernel(h, mlp_forward_kernel<T>, h->grid, MLP_THREADS, sizeof(MlpSmem<T>), mlp_fwd_args<T>(h, u0, p, saved, status));
    };
    return h->cfg.dtype != B200ADJ_F64 ? go(float{}) : go(double{});
}
int mlp_reverse_dispatch(Handle* h, const void* dLdu, void* du0, void* dp) {
    return with_flag(h->cfg.sensealg == B200ADJ_SA_GAUSS, [&](auto GAUSS) { return with_cost(h, [&](auto COST) {
        if (is_mlp_tc(h)) {
            int grid, rc = mlp_tc_launch(h, mlp_tc_reverse_kernel<COST.value, GAUSS.value>, mlp_tcw_reverse_kernel<COST.value, GAUSS.value>,
                                         mlp_rev_args<float>(h, dLdu, du0, dp), grid);
            return rc ? rc : mlp_reduce<float>(h, dp, grid);
        }
        auto go = [&](auto t) {
            using T = decltype(t);
            const int rc = launch_kernel(h, mlp_reverse_kernel<T, COST.value, GAUSS.value>, h->grid, MLP_THREADS, sizeof(MlpSmem<T>),
                                         mlp_rev_args<T>(h, dLdu, du0, dp));
            return rc ? rc : mlp_reduce<T>(h, dp, h->grid);
        };
        return h->cfg.dtype != B200ADJ_F64 ? go(float{}) : go(double{});
    }); });
}
}  // namespace b200adj
