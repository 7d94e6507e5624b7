// ob_lookback.cuh -- the decoupled look-back of the one-launch compactions: K3 (ob_dewarp_frame.cu) and the map-row
// ingest (ob_map_rows.cu).  CTAs take their logical index from a ticket counter, so a CTA's predecessors are always
// running (or done) when it waits for them; each publishes its aggregate, then its inclusive prefix.
#pragma once
#include <cstdint>

#include "ob_arith.cuh"

namespace ob {

__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Per logical CTA a state word (0 = nothing yet, 1 = aggregate published, 2 = inclusive prefix published) and the
// two values; the state words start zeroed.
struct Lookback {
    uint32_t* state;
    unsigned long long* agg;
    unsigned long long* incl;
};

// Called by all 32 lanes of one warp of logical CTA `bid` with the CTA's aggregate: publishes it, looks back over the
// predecessors (one warp looks at 32 of them at a time) and publishes the inclusive prefix.  Returns the exclusive
// prefix in every lane.
__device__ __forceinline__ unsigned long long lookback_exclusive(const Lookback& sc, unsigned bid,
                                                                 unsigned long long aggregate, unsigned lane) {
    if (lane == 0) {
        if (bid == 0) {
            sc.incl[0] = aggregate;
            st_release_u32(&sc.state[0], 2u);
        } else {
            sc.agg[bid] = aggregate;
            st_release_u32(&sc.state[bid], 1u);
        }
    }
    unsigned long long excl = 0;
    if (bid == 0) return excl;
    int p = static_cast<int>(bid) - 1;
    for (;;) {
        const int idx = p - static_cast<int>(lane);
        uint32_t st = 2u;  // positions before CTA 0 behave like a published prefix of zero
        unsigned long long v = 0;
        if (idx >= 0) {
            do {
                st = ld_acquire_u32(&sc.state[idx]);
            } while (st == 0u);
            v = __ldcg(st == 2u ? &sc.incl[idx] : &sc.agg[idx]);
        }
        const unsigned pm = __ballot_sync(0xffffffffu, st == 2u);
        if (pm != 0u) {  // nearest predecessor with an inclusive prefix closes the chain
            const unsigned fl = __ffs(pm) - 1u;
            excl += warp_sum_u64(lane <= fl ? v : 0ull);
            break;
        }
        excl += warp_sum_u64(v);
        p -= 32;
    }
    if (lane == 0) {
        sc.incl[bid] = excl + aggregate;
        st_release_u32(&sc.state[bid], 2u);
    }
    return excl;
}

}  // namespace ob
