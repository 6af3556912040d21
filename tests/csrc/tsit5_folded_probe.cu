// tsit5_folded_probe.cu -- exposes the folded Hermite point table of the fixed-step Tsit5 reverse pass (api.cu,
// build_hermite_folded: OdeRevArgsT::hHf) to the CPU tests, with the 7 theta it is built at (hermite_thetas) and the
// fp32 weights the fp32 reverse pass receives (build_hermite_weights_f32).
#include "handle.h"

// hHf of step h (7 x 4 doubles)
extern "C" void probe_hermite_folded(double h, double* out) {
    b200adj::build_hermite_folded(h, reinterpret_cast<double (*)[4]>(out));
}

// the theta of rows 0..6 (7 doubles)
extern "C" void probe_hermite_thetas(double* out) { b200adj::hermite_thetas(out); }

// OdeRevArgsT<float>::hC4u (7 floats) and hHf (7 x 4 floats) of step h
extern "C" void probe_hermite_weights_f32(double h, float* c4u, float* hf) {
    b200adj::build_hermite_weights_f32(h, c4u, reinterpret_cast<float (*)[4]>(hf));
}
