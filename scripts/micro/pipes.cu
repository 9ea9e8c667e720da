// Micro-benchmark: issue rate of IDP.4A, FFMA, FADD, LOP3 and IMMA.16832.S8 on sm_90a (per SM per clock).
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
template <int OP> __global__ void k(int iters, int * out, long long * cyc) {
    int a[8], b = threadIdx.x * 0x01010101, c = blockIdx.x;
    float f[8];
    for (int i = 0; i < 8; i++) { a[i] = threadIdx.x + i; f[i] = threadIdx.x * 0.5f + i; }
    int d0[4] = {0,0,0,0}, d1[4] = {0,0,0,0}, d2[4]={0,0,0,0}, d3[4]={0,0,0,0};
    long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
        #pragma unroll
        for (int i = 0; i < 8; i++) {
            if (OP == 0) a[i] = __dp4a(a[i], b, c);
            if (OP == 1) f[i] = __fmaf_rn(f[i], 1.0001f, 0.5f);
            if (OP == 2) f[i] = __fadd_rn(f[i], 12582912.f);
            if (OP == 3) a[i] = (a[i] << 4) & 0xF0F0F0F0;
            if (OP == 5) f[i] = __fmaf_rn(f[i], f[(i+1)&7], f[(i+3)&7]);
        }
        if (OP == 4) {
            asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                : "+r"(d0[0]), "+r"(d0[1]), "+r"(d0[2]), "+r"(d0[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]));
            asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                : "+r"(d1[0]), "+r"(d1[1]), "+r"(d1[2]), "+r"(d1[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]));
            asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                : "+r"(d2[0]), "+r"(d2[1]), "+r"(d2[2]), "+r"(d2[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]));
            asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                : "+r"(d3[0]), "+r"(d3[1]), "+r"(d3[2]), "+r"(d3[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]));
        }
    }
    long long t1 = clock64();
    int s = 0; for (int i = 0; i < 8; i++) s += a[i] + (int) f[i];
    for (int i = 0; i < 4; i++) s += d0[i] + d1[i] + d2[i] + d3[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
template <int OP> void run(const char * name, int per_iter) {
    int * out; long long * cyc; cudaMalloc(&out, 132 * 1024 * 4); cudaMalloc(&cyc, 132 * 8);
    for (int warps : {4, 8, 16, 32}) {
        const int iters = 2000;
        k<OP><<<132, warps * 32>>>(iters, out, cyc); cudaDeviceSynchronize();
        k<OP><<<132, warps * 32>>>(iters, out, cyc); cudaDeviceSynchronize();
        long long h[132]; cudaMemcpy(h, cyc, sizeof h, cudaMemcpyDeviceToHost);
        double c = 0; for (int i = 0; i < 132; i++) c += h[i]; c /= 132;
        printf("%-8s warps/SM %2d : %.2f warp-instr/clk/SM (%.2f per SMSP)\n", name, warps, (double) iters * per_iter * warps / c, (double) iters * per_iter * warps / c / 4);
    }
}
int main() {
    run<0>("IDP.4A", 8); run<1>("FFMA.imm", 8); run<5>("FFMA.rrr", 8); run<2>("FADD", 8); run<3>("SHL+LOP", 16); run<4>("IMMA", 4);
    return 0;
}
