// tsit5_tables_probe.cu -- exposes the step-size-scaled Tsit5 tables libb200adj builds for a handle (api.cu,
// build_tsit5_tables) to the CPU tests: the table struct is copied out as a flat array of doubles (or floats, as
// cast_tables hands it to the fp32 kernels), with the c4-from-du weights (build_c4_du_weights) and the dense-output
// polynomials (tsit5_weights) that the fixed-step reverse pass receives next to it.
#include "handle.h"

extern "C" int probe_tsit5_tables(double h, double* out, int cap) {
    static_assert(sizeof(b200adj::Tsit5Tables) % sizeof(double) == 0, "Tsit5Tables holds doubles only");
    const int n = (int)(sizeof(b200adj::Tsit5Tables) / sizeof(double));
    if (n > cap) return -n;
    b200adj::Tsit5Tables t;
    b200adj::build_tsit5_tables(h, &t);
    memcpy(out, &t, sizeof(t));
    return n;
}

// the same tables after cast_tables, as the fp32 forward and reverse kernels receive them
extern "C" int probe_tsit5_tables_f32(double h, float* out, int cap) {
    static_assert(sizeof(b200adj::Tsit5TablesT<float>) % sizeof(float) == 0, "Tsit5TablesT<float> holds floats only");
    const int n = (int)(sizeof(b200adj::Tsit5TablesT<float>) / sizeof(float));
    if (n > cap) return -n;
    b200adj::Tsit5Tables t;
    b200adj::build_tsit5_tables(h, &t);
    b200adj::Tsit5TablesT<float> f;
    b200adj::cast_tables(t, &f);
    memcpy(out, &f, sizeof(f));
    return n;
}

// OdeRevArgsT::hC4u of step h (7 doubles)
extern "C" void probe_c4_du_weights(double h, double* out) { b200adj::build_c4_du_weights(h, out); }

// OdeRevArgsT::Rpoly: b_j(theta) = sum_m R[j][m] theta^(m+1) (7 x 4 doubles)
extern "C" void probe_tsit5_rpoly(double* out) { b200adj::tsit5_weights(0.0, nullptr, reinterpret_cast<double (*)[4]>(out)); }
