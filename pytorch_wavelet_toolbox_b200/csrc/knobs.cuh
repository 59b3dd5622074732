// knobs.cuh -- tuning / test switches of libwtb200, read from the environment ONCE (WTB200_<NAME>) when the
// library is first used and changeable at run time through wt_set_knob() (include/wtb200.h).  No getenv()
// on any transform call.
#pragma once

#include <atomic>
#include <climits>
#include <cstdlib>
#include <cstring>

namespace wtb {

// Matrix FWT (matrix_dmma.cuh, matrix_fused.cuh):
//   NO_DMMA          float64 without the FP64 tensor-core cascades (scalar fused analysis, per-level synthesis)
//   MATF_K / MATI_K  levels per launch (analysis / float64 synthesis);  MATF_KCOARSE the same for rows <= 8192 samples
//   MATF_CHUNK / MATI_CHUNK   finest-level samples per CTA;  MATF_NT / MATI_NT  threads per CTA (128 | 256)
//   MATF_CPC         scalar fused analysis: consecutive chunks one CTA streams
//   MATI_MINCTAS, MATI_MERGE_N   short rows: halve the chunk below this CTA count / merge levels of rows <= N
#define WTB_KNOB_LIST(X)                                                                                     \
    X(DISABLE_FUSED) X(NO_FFMA2) X(CHUNK) X(STREAMS) X(FWD3D_TILE) X(CONVF_CHUNK) X(CONVF_K) X(MATF_CHUNK)     \
    X(MATI_CHUNK) X(MATF_K) X(MATI_K) X(MATI_NT) X(MATI_MINCTAS) X(MATI_MERGE_N)                               \
    X(MATF_KCOARSE) X(NO_WPAIR) X(WPAIR_SEG) X(WPAIR_MIN) X(WPAIR_DEEP)                                            \
    X(NO_AUX_STREAM) X(WPAIR_VAR) X(WPAIR) X(MATF_NT) X(MATF_MINB) X(MATF_CPC) X(NO_DMMA) X(FUSE2)

enum KnobId {
#define X(n) K_##n,
    WTB_KNOB_LIST(X)
#undef X
    K_COUNT
};

static const char* const kKnobNames[K_COUNT] = {
#define X(n) #n,
    WTB_KNOB_LIST(X)
#undef X
};

constexpr long long KNOB_UNSET = LLONG_MIN;

struct KnobTable {
    std::atomic<long long> v[K_COUNT];
    KnobTable() {
        for (int k = 0; k < K_COUNT; ++k) {
            char name[64] = "WTB200_";
            strncat(name, kKnobNames[k], sizeof(name) - 8);
            const char* ev = getenv(name);
            long long val = KNOB_UNSET;
            if (ev) {
                char* end = nullptr;
                val = strtoll(ev, &end, 10);
                if (end == ev) val = 1;   // set, but not a number: a plain switch
            }
            v[k].store(val, std::memory_order_relaxed);
        }
    }
};

static inline KnobTable& knob_table() {
    static KnobTable t;
    return t;
}
static inline bool knob_is_set(KnobId k) { return knob_table().v[k].load(std::memory_order_relaxed) != KNOB_UNSET; }
static inline bool knob_on(KnobId k) {
    const long long v = knob_table().v[k].load(std::memory_order_relaxed);
    return v != KNOB_UNSET && v != 0;
}
static inline long long knob_val(KnobId k, long long dflt) {
    const long long v = knob_table().v[k].load(std::memory_order_relaxed);
    return v == KNOB_UNSET ? dflt : v;
}
static inline int knob_find(const char* name) {
    if (!name) return -1;
    if (!strncmp(name, "WTB200_", 7)) name += 7;
    for (int k = 0; k < K_COUNT; ++k)
        if (!strcmp(name, kKnobNames[k])) return k;
    return -1;
}

}  // namespace wtb
