// peer_sync.cuh -- the flag primitives of the NVLink peer-memory exchanges (peer_gather.cu, grad_exchange.cu, bn.cu).
//
// A producer stores its data into the peer's symmetric buffer, runs __threadfence_system() and then publishes a replay
// number with st_release_sys; a consumer spins with ld_acquire_sys until the number arrives and then reads the data with
// __ldcg (written by another GPU: not through L1).  A spin that lasts kPeerSpinLimit cycles gives up: the caller counts
// it, so a rank that died cannot hang the others' GPUs.
#pragma once

namespace ssd3d {

constexpr long long kPeerSpinLimit = 1LL << 33;        // ~4 s of clock64 at H100 clocks

__device__ __forceinline__ int ld_acquire_sys(const int *p)
{
    int v;
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ void st_release_sys(int *p, int v)
{
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

}  // namespace ssd3d
