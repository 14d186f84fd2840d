// Pipe-throughput probe for the instructions of the SW inner loop (sm_90a).  Prints warp-instructions
// per cycle per SM for independent chains, 32 warps per SM.  Design aid, not part of the product.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

template <int OP>
__global__ void __launch_bounds__(1024, 1) k(uint32_t* out, int iters, long long* cyc)
{
    uint32_t x[8], y = threadIdx.x * 2654435761u, z = blockIdx.x + 12345u;
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = y + i * 77u;
    __shared__ uint4 sm[1024];
    sm[threadIdx.x] = make_uint4(y, z, y ^ z, 1);
    __syncthreads();
    long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (OP == 0) x[i] = __viaddmax_s16x2(x[i], 0xFFFFFFFFu, y);
            if (OP == 1) x[i] = __vimax3_s16x2(x[i], y, z);
            if (OP == 2) x[i] = __vadd2(x[i], 0xFFFAFFFAu);
            if (OP == 3) x[i] = __vimax3_s16x2_relu(x[i], y, z);
            if (OP == 4) x[i] = x[i] * 3u + y;
            if (OP == 5) { x[i] = __viaddmax_s16x2(x[i], 0xFFFFFFFFu, y); if (i & 1) z = z * 5u + x[i]; }
            if (OP == 6) x[i] = __shfl_up_sync(0xffffffffu, x[i], 1, 8);
            if (OP == 7) { uint4 v = sm[(threadIdx.x + x[i]) & 1023]; x[i] = v.x + v.y + v.z + v.w; }
            if (OP == 8) x[i] = __viaddmax_s16x2_relu(x[i], y, z);
            if (OP == 9) { x[i] = __viaddmax_s16x2(x[i], 0xFFFFFFFFu, y); asm volatile("mov.b32 %0, %1;" : "=r"(z) : "r"(x[i])); }
            if (OP == 10) x[i] = (x[i] + y) ^ z;       // IADD3/LOP3 (alu)
            if (OP == 11) x[i] = __byte_perm(x[i], y, 0x7610);                       // PRMT
            if (OP == 12) { x[i] = __viaddmax_s16x2(x[i], 0xFFFFFFFFu, y); z = __byte_perm(z, x[i], 0x7610); }   // DPX + PRMT 1:1
            if (OP == 13) { x[i] = __viaddmax_s16x2(x[i], 0xFFFFFFFFu, y); z = (z ^ x[i]) | 0x80008000u; }       // DPX + LOP3 1:1
            if (OP == 14) { x[i] = __viaddmax_s16x2(x[i], 0xFFFFFFFFu, y); z = (z & x[i]) + 0x10001u; y = y ^ (z >> 3); }  // DPX + 3 alu
            if (OP == 15) x[i] = __vcmpeq2(x[i], y) + z;                             // packed compare (emulated?)
            if (OP == 16) x[i] = max((int)x[i], (int)y) + 1;                         // 32-bit max
            // which DPX instructions share an issue resource?  independent chains, alternating kinds
            if (OP == 17) x[i] = (i & 1) ? __viaddmax_s16x2(x[i], 0xFFFFFFFFu, y) : __vimax3_s16x2(x[i], y, z);
            if (OP == 18) x[i] = (i & 1) ? __viaddmax_s16x2(x[i], 0xFFFFFFFFu, y) : __vmaxs2(x[i], y);
            if (OP == 19) x[i] = (i & 1) ? __vimax3_s16x2(x[i], y, z) : __vmaxs2(x[i], y);
            if (OP == 20) x[i] = __vmaxs2(x[i], y);
            if (OP == 21) x[i] = (i & 1) ? __viaddmax_s16x2(x[i], 0xFFFFFFFFu, y) : x[i] + 0xFFFAFFFAu;
            if (OP == 22) x[i] = (i & 1) ? __vimax3_s16x2(x[i], y, z) : x[i] + 0xFFFAFFFAu;
            if (OP == 23) x[i] = (i % 3 == 0) ? __viaddmax_s16x2(x[i], 0xFFFFFFFFu, y) : (i % 3 == 1) ? __vimax3_s16x2(x[i], y, z) : x[i] + 0xFFFAFFFAu;
            if (OP == 24) x[i] = (i & 1) ? __viaddmax_s16x2(x[i], 0xFFFFFFFFu, y) : __viaddmax_s16x2_relu(x[i], y, z);
        }
    }
    long long t1 = clock64();
    uint32_t s = z;
#pragma unroll
    for (int i = 0; i < 8; ++i) s ^= x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int OP> void run(const char* name, int per_iter)
{
    int n_sm = 0; cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, 0);
    uint32_t* out; long long* cyc; cudaMalloc(&out, n_sm * 1024 * 4); cudaMalloc(&cyc, n_sm * 8);
    const int iters = 4096;
    k<OP><<<n_sm, 1024>>>(out, 64, cyc);
    k<OP><<<n_sm, 1024>>>(out, iters, cyc);
    cudaDeviceSynchronize();
    long long h[256]; cudaMemcpy(h, cyc, n_sm * 8, cudaMemcpyDeviceToHost);
    double avg = 0; for (int i = 0; i < n_sm; ++i) avg += h[i]; avg /= n_sm;
    printf("%-44s %7.3f warp-instr/cycle/SM  (%.1f cycles per warp-instr per SMSP)\n", name, 32.0 * iters * per_iter / avg,
           avg / (8.0 * iters * per_iter));
    cudaFree(out); cudaFree(cyc);
}

int main()
{
    run<0>("VIADDMNMX.S16x2", 8);
    run<8>("VIADDMNMX.S16x2.RELU", 8);
    run<1>("VIMNMX3.S16x2", 8);
    run<3>("VIMNMX3.S16x2.RELU", 8);
    run<2>("VIADD.16x2", 8);
    run<10>("IADD3+LOP3 (2 per slot)", 16);
    run<4>("IMAD", 8);
    run<5>("VIADDMNMX + IMAD 2:1 (12 per iter)", 12);
    run<9>("VIADDMNMX + MOV 1:1 (16 per iter)", 16);
    run<11>("PRMT", 8);
    run<12>("VIADDMNMX + PRMT 1:1 (16 per iter)", 16);
    run<13>("VIADDMNMX + LOP3 1:1 (16 per iter)", 16);
    run<14>("VIADDMNMX + 3-4 int ops (per DPX)", 8);
    run<15>("__vcmpeq2 (+IADD)", 8);
    run<16>("IMNMX.S32 (+IADD)", 8);
    run<20>("VIMNMX.S16x2 (2-input)", 8);
    run<17>("VIADDMNMX + VIMNMX3 1:1", 8);
    run<18>("VIADDMNMX + VIMNMX 1:1", 8);
    run<19>("VIMNMX3 + VIMNMX 1:1", 8);
    run<21>("VIADDMNMX + plain add 1:1", 8);
    run<22>("VIMNMX3 + plain add 1:1", 8);
    run<23>("VIADDMNMX + VIMNMX3 + plain add 3:3:2", 8);
    run<24>("VIADDMNMX + VIADDMNMX.RELU 1:1", 8);
    run<6>("SHFL.UP", 8);
    run<7>("LDS.128 (+3 IADD)", 8);
    return 0;
}
