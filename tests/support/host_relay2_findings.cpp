// TEST AID ONLY: the emulated bulk kernels of host_relay2_sliced.cpp, plus a look at the findings scratch (SegPlan[max_streams])
// between launch sets.  Never linked into the product library.
#include "host_relay2_sliced.cpp"

extern "C" {

// bytes of the findings scratch that are not zero: k_commit2 leaves none behind
uint64_t lgwt_bulk_findings_nonzero(void* h) {
    HostEngine* e = (HostEngine*)h;
    const uint8_t* p = (const uint8_t*)e->plan.data();
    uint64_t n = 0;
    for (size_t i = 0; i < e->plan.size() * sizeof(SegPlan); ++i) n += p[i] != 0;
    return n;
}

}  // extern "C"
