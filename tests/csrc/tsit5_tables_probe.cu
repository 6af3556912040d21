// tsit5_tables_probe.cu -- exposes the step-size-scaled Tsit5 tables libb200adj builds for a handle (api.cu,
// build_tsit5_tables) to the CPU tests: the table struct is copied out as a flat array of doubles.
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
