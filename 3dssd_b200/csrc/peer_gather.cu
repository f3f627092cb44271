// peer_gather.cu -- the per-step exchange of the sharded path (SURVEY.md section 8e) as ONE kernel over NVLink peer memory.
//
// The reference has no multi-GPU inference (lib/core/evaluator.py:145-147 runs one GPU, batch 1); the sharded step of
// this repo ends with an all-gather of the per-scene detection block every rank's NMS produced (3dssd_b200/dist.py).
// ncclAllGather does that correctly, but captured into 8-24 concurrently replayed step graphs it adds a per-step cost
// that a one-GPU step does not have.  The exchange is 3.6 KB per scene: all it needs is  store my slice into every peer's buffer -> publish a flag -> wait for the peers' flags.
//
// Buffers (3dssd_b200/dist.py PeerGather): every rank owns a SYMMETRIC allocation, mapped into all peers
// (torch.distributed._symmetric_memory: cuMem + fabric / fd handles), holding for each of two parities a receive area
// of `world` slices and `world` flag words.  Replay number s (counted on the device, so a captured launch needs no
// changing argument) uses parity s & 1:
//     CTA p:  copy my slice -> peer p's receive area [parity][my rank]          (16-byte stores over NVLink; p == rank: local)
//             __threadfence_system(); st.release.sys  peer p's flag[parity][my rank] = s
//             spin ld.acquire.sys on MY flag[parity][p] until it reads >= s      (peer p has delivered replay s)
//             copy MY receive area [parity][p] -> out[p]                          (plain local result buffer, L1 bypassed)
// Two parities are what makes overwriting safe without an acknowledgement: a peer can start replay s+2 (which reuses the
// parity of s) only after its wait of replay s+1 saw MY flag of s+1, and I publish s+1 only after my kernel of replay s --
// copy-out included -- has finished (same stream).  Every rank must call the exchange the same number of times.  A wait
// that lasts ~4 s gives up and counts itself in state[2] (a rank that died must not hang the others' GPUs).
#include "common.cuh"

namespace ssd3d {

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

struct PeerGatherParams {
    const uint4 *src;          // my slice (slice_bytes, 16-byte multiple)
    uint8_t *const *peer_base; // DEVICE array [world]: base of every rank's symmetric allocation as mapped here
    uint4 *out;                // [world][slice_bytes] local result
    int *state;                // [0] replays done so far, [1] CTAs of the current replay that have finished, [2] time-outs
    size_t slice_bytes, recv_off[2], flag_off[2];
    int world, rank;
};

__global__ void __launch_bounds__(256)
peer_allgather_kernel(const PeerGatherParams p)
{
    const int peer = blockIdx.x, tid = threadIdx.x;
    __shared__ int s_seq;
    if (tid == 0) s_seq = *reinterpret_cast<volatile int *>(p.state) + 1;   // state[0] changes only after every CTA has read it
    __syncthreads();
    const int seq = s_seq, par = seq & 1;
    const size_t n16 = p.slice_bytes / 16;
    uint8_t *theirs = p.peer_base[peer], *mine = p.peer_base[p.rank];
    uint4 *dst = reinterpret_cast<uint4 *>(theirs + p.recv_off[par] + (size_t)p.rank * p.slice_bytes);
    for (size_t i = tid; i < n16; i += blockDim.x) dst[i] = p.src[i];
    __threadfence_system();
    __syncthreads();
    if (tid == 0) {
        st_release_sys(reinterpret_cast<int *>(theirs + p.flag_off[par]) + p.rank, seq);
        const int *flag = reinterpret_cast<const int *>(mine + p.flag_off[par]) + peer;
        const long long t0 = clock64();
        while (ld_acquire_sys(flag) < seq) {
            if (clock64() - t0 > (1LL << 33)) { atomicAdd(p.state + 2, 1); break; }   // ~4 s: a peer never came (counted, not hung)
        }
    }
    __syncthreads();
    const uint4 *got = reinterpret_cast<const uint4 *>(mine + p.recv_off[par] + (size_t)peer * p.slice_bytes);
    uint4 *res = p.out + (size_t)peer * n16;
    for (size_t i = tid; i < n16; i += blockDim.x) res[i] = __ldcg(got + i);       // written by another GPU: not through L1
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        if (atomicAdd(p.state + 1, 1) == p.world - 1) {            // last CTA of this replay: publish the new count
            p.state[1] = 0;
            __threadfence();
            *reinterpret_cast<volatile int *>(p.state) = seq;
        }
    }
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" int ssd3d_peer_allgather(const void *src, size_t slice_bytes, void *const *peer_base, int world, int rank,
                                    size_t recv_off0, size_t recv_off1, size_t flag_off0, size_t flag_off1, int *state,
                                    void *out, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(world >= 1 && world <= 64 && rank >= 0 && rank < world, "peer_allgather: bad world=%d rank=%d", world, rank);
    SSD3D_REQUIRE(src && peer_base && state && out, "peer_allgather: null pointer");
    SSD3D_REQUIRE(slice_bytes > 0 && slice_bytes % 16 == 0 && recv_off0 % 16 == 0 && recv_off1 % 16 == 0 && flag_off0 % 4 == 0 &&
                  flag_off1 % 4 == 0, "peer_allgather: slice / offsets must be 16-byte (flags 4-byte) multiples");
    SSD3D_REQUIRE(((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0, "peer_allgather: buffers must be 16-byte aligned");
    PeerGatherParams p = {};
    p.src = (const uint4 *)src; p.peer_base = (uint8_t *const *)peer_base; p.out = (uint4 *)out; p.state = state;
    p.slice_bytes = slice_bytes; p.recv_off[0] = recv_off0; p.recv_off[1] = recv_off1; p.flag_off[0] = flag_off0; p.flag_off[1] = flag_off1;
    p.world = world; p.rank = rank;
    peer_allgather_kernel<<<world, 256, 0, (cudaStream_t)stream>>>(p);
    SSD3D_LAUNCH_CHECK("peer_allgather_kernel");
}
