// Dependent-chain latencies (cycles per operation, one warp unless noted) of the warp-collective and control operations the
// pruned FPS round is made of (csrc/fps_bucket.cu): the numbers a redesign of that round has to be priced with.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench/warp_ops tools/ubench/warp_ops.cu && tools/ubench/warp_ops
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int ITERS = 2048;

__device__ __forceinline__ long long now() { return clock64(); }

template <int OP>
__global__ void __launch_bounds__(512, 1) chain(double *out, unsigned seed)
{
    __shared__ unsigned sm[1024];
    const int lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) sm[i] = (i * 37u + 11u) & 1023u;
    __syncthreads();
    unsigned v = seed + threadIdx.x, w = seed ^ 0x55u;
    float f = (float)v;
    float dist[32];
#pragma unroll
    for (int i = 0; i < 32; i++) dist[i] = (float)(i + seed);
    const long long t0 = now();
    for (int it = 0; it < ITERS; it++) {
        if (OP == 0) v = __reduce_max_sync(0xffffffffu, v ^ lane) + 1u;                       // REDUX / CREDUX
        if (OP == 1) v = __ballot_sync(0xffffffffu, (v >> lane) & 1u) + it;                   // VOTE
        if (OP == 2) v = __shfl_sync(0xffffffffu, v, (v + 1) & 31) + 1u;                      // SHFL.IDX
        if (OP == 3) v = sm[v & 1023u];                                                       // LDS pointer chase
        if (OP == 4) { __syncthreads(); v += 1u; }                                            // BAR.SYNC, 16 warps
        if (OP == 5) v = (unsigned)__ffs(v | 0x80000000u) + (v >> 1);                         // BREV + FLO
        if (OP == 6) f = fmaf(f, 1.0000001f, 1.0f);                                           // FFMA
        if (OP == 7) {                                                                        // one full (value, key) arg-max stage
            const unsigned mx = __reduce_max_sync(0xffffffffu, v ^ lane);
            const unsigned km = __reduce_min_sync(0xffffffffu, ((v ^ lane) == mx) ? (w + lane) : 0x7fffffffu);
            const unsigned bal = __ballot_sync(0xffffffffu, (v ^ lane) == mx && (w + lane) == km);
            v = mx + (unsigned)__ffs(bal) + km;
        }
        if (OP == 8) {                                                                        // warp-uniform 32-way switch on registers
            const int i = (int)(__shfl_sync(0xffffffffu, v, 0) & 31u);
            float nd;
            switch (i) {
#define C(I) case I: nd = fminf(f, dist[I]); dist[I] = nd + 1.0f; break;
                C(0) C(1) C(2) C(3) C(4) C(5) C(6) C(7) C(8) C(9) C(10) C(11) C(12) C(13) C(14) C(15)
                C(16) C(17) C(18) C(19) C(20) C(21) C(22) C(23) C(24) C(25) C(26) C(27) C(28) C(29) C(30)
                default: nd = fminf(f, dist[31]); dist[31] = nd + 1.0f; break;
#undef C
            }
            v = v * 1664525u + 1013904223u + (unsigned)nd;
        }
        if (OP == 9) {                                                                        // the SHFL of OP 8 alone (to subtract)
            const int i = (int)(__shfl_sync(0xffffffffu, v, 0) & 31u);
            v = v * 1664525u + 1013904223u + (unsigned)i;
        }
    }
    const long long t1 = now();
    float acc = f;
#pragma unroll
    for (int i = 0; i < 32; i++) acc += dist[i];
    if (threadIdx.x == 0) out[OP] = (double)(t1 - t0) / ITERS;
    if (v == 0xdeadbeefu && acc == 1.0f) out[63] = 1.0;                                       // keep everything alive
}

int main()
{
    double *d, h[64] = {0};
    cudaMalloc(&d, sizeof(h));
    cudaMemset(d, 0, sizeof(h));
    const char *names[10] = {"redux_max_u32", "vote_ballot", "shfl_idx", "lds_chase", "bar_sync_512_threads", "ffs(brev+flo)", "ffma",
                             "argmax_stage(redux+redux+ballot+ffs)", "uniform_switch32_on_registers(+shfl)", "shfl+lcg (baseline of the switch)"};
#define RUN(OP, T) chain<OP><<<1, T>>>(d, 12345u)
    for (int rep = 0; rep < 2; rep++) {
        RUN(0, 32); RUN(1, 32); RUN(2, 32); RUN(3, 32); RUN(4, 512); RUN(5, 32); RUN(6, 32); RUN(7, 32); RUN(8, 32); RUN(9, 32);
        cudaDeviceSynchronize();
    }
    cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost);
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    printf("{\"gpu\": \"%s\", \"unit\": \"cycles per dependent operation (clock64, %d iterations)\"", p.name, ITERS);
    for (int i = 0; i < 10; i++) printf(",\n \"%s\": %.1f", names[i], h[i]);
    printf("}\n");
    return cudaGetLastError() != cudaSuccess;
}
