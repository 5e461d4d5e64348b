// Calibration micro-benchmark: cost of N scattered 32-bit reductions / CAS / 128-bit CAS / 32-byte gathers with the
// access pattern of the association kernel (mostly consecutive targets with gaps).   nvcc -arch=sm_90a -O3 -o ab atomics_bench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
struct __align__(16) U128 { unsigned long long lo, hi; };
__device__ __forceinline__ U128 cas128(U128 *addr, U128 e, U128 d) {
  U128 o;
  asm volatile("{\n\t.reg .b128 e, d, o;\n\tmov.b128 e, {%2, %3};\n\tmov.b128 d, {%4, %5};\n\t"
               "atom.global.relaxed.gpu.cas.b128 o, [%6], e, d;\n\tmov.b128 {%0, %1}, o;\n\t}"
               : "=l"(o.lo), "=l"(o.hi) : "l"(e.lo), "l"(e.hi), "l"(d.lo), "l"(d.hi), "l"(addr) : "memory");
  return o;
}
__device__ __forceinline__ unsigned target(unsigned i, unsigned P, int mode) {
  if (mode == 0) return (i + (i >> 5) * 3u) % P;                      // coherent: consecutive with gaps
  unsigned x = i * 2654435761u; x ^= x >> 15; x *= 2246822519u; x ^= x >> 13;  // random
  return x % P;
}
template <int OP>
__global__ void k(unsigned *slot, U128 *rec, const float4 *frec, float4 *sink, unsigned n, unsigned P, int mode) {
  unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned t = target(i, P, mode);
  if (OP == 0) atomicMax(slot + t, i + 1);                      // RED.32
  if (OP == 1) { unsigned o = atomicCAS(slot + t, 0u, i + 1); if (o == 12345u) sink[0].x = 1.f; }  // CAS.32 with return
  if (OP == 2) { U128 o = cas128(rec + t, U128{0, 0}, U128{i, i}); if (o.lo == 12345u) sink[0].x = 1.f; }
  if (OP == 3) { float4 a = frec[2 * (size_t)t], b = frec[2 * (size_t)t + 1]; if (a.x + b.y == 12345.f) sink[0] = a; }  // 32 B gather
  if (OP == 4) slot[t] = i + 1;                                 // plain store
}
int main() {
  const unsigned P = 8 * 307200, n = 2300000, ng = 4000000;
  unsigned *slot; U128 *rec; float4 *frec, *sink; char *flush;
  cudaMalloc(&slot, P * 4); cudaMalloc(&rec, (size_t)P * 16); cudaMalloc(&frec, (size_t)P * 32); cudaMalloc(&sink, 64);
  cudaMalloc(&flush, 256 << 20);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const char *names[] = {"RED.MAX.32", "CAS.32+ret", "CAS.128+ret", "gather 32B", "store 32"};
  for (int warm = 0; warm < 2; ++warm)
    for (int mode = 0; mode < 2; ++mode)
      for (int resident = 0; resident < 2; ++resident)
        for (int op = 0; op < 5; ++op) {
          unsigned cnt = op == 3 ? ng : n;
          cudaMemset(slot, 0, P * 4); cudaMemset(rec, 0, (size_t)P * 16);
          if (!resident) cudaMemset(flush, 1, 256 << 20);  // evict the targets from L2
          else if (op == 3) cudaMemset(frec, 0, (size_t)P * 32);
          cudaEventRecord(e0);
          dim3 g((cnt + 255) / 256);
          if (op == 0) k<0><<<g, 256>>>(slot, rec, frec, sink, cnt, P, mode);
          if (op == 1) k<1><<<g, 256>>>(slot, rec, frec, sink, cnt, P, mode);
          if (op == 2) k<2><<<g, 256>>>(slot, rec, frec, sink, cnt, P, mode);
          if (op == 3) k<3><<<g, 256>>>(slot, rec, frec, sink, cnt, P, mode);
          if (op == 4) k<4><<<g, 256>>>(slot, rec, frec, sink, cnt, P, mode);
          cudaEventRecord(e1); cudaEventSynchronize(e1);
          float ms; cudaEventElapsedTime(&ms, e0, e1);
          if (warm) printf("%-12s %-8s %-12s n=%u  %.1f us  (%.1f ps/op)\n", names[op], mode ? "random" : "coherent",
                           resident ? "L2-warm" : "L2-flushed", cnt, ms * 1e3, ms * 1e9 / cnt);
        }
  return 0;
}
