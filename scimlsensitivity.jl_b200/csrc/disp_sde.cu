// disp_sde.cu -- SDE kernels (disp_sde.inc) instantiated for the built-in families SdeLotkaVolterra and SdeLinear2, and
// the noise export kernel
#include "disp_sde.inc"
namespace b200adj {
template int launch_sde_fwd<SdeLotkaVolterra>(Handle*, const SdeFwdArgs&);
template int launch_sde_rev<SdeLotkaVolterra>(Handle*, const SdeRevArgs&);
template int launch_sde_fwd<SdeLinear2>(Handle*, const SdeFwdArgs&);
template int launch_sde_rev<SdeLinear2>(Handle*, const SdeRevArgs&);

int sde_noise_launch(Handle* h, const SdeNoiseArgs& a, int64_t total) {
    return launch_kernel(h, sde_noise_kernel<0>, (unsigned)((total + 255) / 256), 256, 0, a);
}
}  // namespace b200adj
