/*
 * mm_issue_peak.cu -- measured INT32 issue peaks of the SM (SURVEY 8(d): "builder must measure that peak with an IMAD
 * micro-benchmark"). K1's per-base loop is two bit-exact Murmur3 evaluations: 32-bit multiply-adds (FMA pipe: IMAD,
 * IMAD.WIDE) and shifts / logic / adds (ALU pipe: SHF, LOP3, IADD3, PRMT). This program times long dependent chains of
 * each instruction (8 independent chains per thread, 1024 threads per SM resident, every SM busy) and of the mixes the
 * hash uses, and prints warp instructions per clock per SM. bench.py reads the JSON line (profiles/issue_peak.json) for
 * the instruction roofline of K1.
 *
 * build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o mm_issue_peak mm_issue_peak.cu
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../mm_hash.h"

#ifndef MM_SASS_ROUND
#define MM_SASS_ROUND 17.6 /* SASS instructions of one OP_HASH_ROUND step / one OP_HASH19 step: counted by the Makefile rule */
#endif
#ifndef MM_SASS_HASH19
#define MM_SASS_HASH19 68.0
#endif
#define CHAINS 8
#define UNROLL 16

enum Op { OP_IMAD, OP_IMAD_WIDE, OP_SHF, OP_LOP3, OP_IADD3, OP_PRMT, OP_MIX_IMAD_LOP3, OP_MIX_IMAD_SHF, OP_MIX_WIDE_SHF,
          OP_MIX_MURMUR, OP_NOWIDE_MIX, OP_WIDE_IMAD, OP_HASH_ROUND, OP_HASH19, OP_COUNT };
static const char *OP_NAME[OP_COUNT] = {"imad", "imad_wide+lop3", "shf", "lop3", "iadd3", "prmt", "imad+lop3", "imad+shf",
                                        "imad_wide+lop3+shf", "murmur_mix(3imad:1wide:2shf:3lop3:1iadd3)",
                                        "same_mix_without_wide(4imad:2shf:3lop3:1iadd3)", "imad_wide+lop3+2imad",
                                        "murmur3_block_half(mm_hash.h: 2 mulc, 2 rotl, xor, x5+c)", "murmur3_x64_128_k19(mm_hash.h, full hash)"};
/* SASS instructions issued per chain per inner step (checked with cuobjdump: one SASS instruction per PTX instruction
 * here; a mad.wide with a 64-bit addend would be split by ptxas into IMAD.WIDE(.., RZ) + IADD3 + IADD3.X, so the wide
 * multiply is measured without an addend, as K1's SASS uses it, and with a LOP3 consuming its high word so that ptxas
 * cannot narrow it to a 32-bit IMAD) */
/* the last two run mm_hash.h's own device code; their SASS instruction counts per step are filled in from cuobjdump */
static const double OP_INSTR[OP_COUNT] = {1, 2, 1, 1, 2, 1, 2, 2, 3, 10, 10, 4, MM_SASS_ROUND, MM_SASS_HASH19};

template <int OP>
__device__ __forceinline__ void step(uint32_t &a, uint32_t &b, uint64_t &w, uint32_t m, uint32_t c)
{
  if (OP == OP_IMAD) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(m), "r"(c));
  if (OP == OP_IMAD_WIDE) { /* multiplicand = low word of the running value: nothing is loop-invariant */
    asm volatile("{ .reg .b32 lo, hi; mov.b64 {lo, hi}, %0; mul.wide.u32 %0, lo, %2; mov.b64 {lo, hi}, %0; lop3.b32 %1, %1, hi, %2, 0x96; }" : "+l"(w), "+r"(a) : "r"(m));
  }
  if (OP == OP_SHF) asm volatile("shf.l.wrap.b32 %0, %0, %1, 13;" : "+r"(a) : "r"(b));
  if (OP == OP_LOP3) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a) : "r"(m), "r"(c));
  if (OP == OP_IADD3) { asm volatile("add.u32 %0, %0, %1;" : "+r"(a) : "r"(b)); asm volatile("add.u32 %0, %0, %1;" : "+r"(b) : "r"(a)); }
  if (OP == OP_PRMT) asm volatile("prmt.b32 %0, %0, %1, 0x4321;" : "+r"(a) : "r"(b));
  if (OP == OP_MIX_IMAD_LOP3) {
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(m), "r"(c));
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(b) : "r"(m), "r"(c));
  }
  if (OP == OP_MIX_IMAD_SHF) {
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(m), "r"(c));
    asm volatile("shf.l.wrap.b32 %0, %0, %1, 13;" : "+r"(b) : "r"(c));
  }
  if (OP == OP_MIX_WIDE_SHF) {
    asm volatile("{ .reg .b32 lo, hi; mov.b64 {lo, hi}, %0; mul.wide.u32 %0, lo, %2; mov.b64 {lo, hi}, %0; lop3.b32 %1, %1, hi, %2, 0x96; }" : "+l"(w), "+r"(a) : "r"(m));
    asm volatile("shf.l.wrap.b32 %0, %0, %1, 13;" : "+r"(b) : "r"(c));
  }
  if (OP == OP_MIX_MURMUR) { /* the instruction mix of one 64-bit multiply + rotate + xor + add of the hash */
    asm volatile("{ .reg .b32 lo, hi; mov.b64 {lo, hi}, %0; mul.wide.u32 %0, lo, %2; mov.b64 {lo, hi}, %0; lop3.b32 %1, %1, hi, %2, 0x96; }" : "+l"(w), "+r"(a) : "r"(m));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(m), "r"(c));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(b) : "r"(m), "r"(c));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(c), "r"(m));
    asm volatile("shf.l.wrap.b32 %0, %0, %1, 31;" : "+r"(a) : "r"(b));
    asm volatile("shf.l.wrap.b32 %0, %0, %1, 31;" : "+r"(b) : "r"(a));
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a) : "r"(m), "r"(c));
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(b) : "r"(m), "r"(c));
    asm volatile("add.u32 %0, %0, %1;" : "+r"(a) : "r"(b));
  }
  if (OP == OP_NOWIDE_MIX) { /* the same mix with the wide multiply replaced by a 32-bit one */
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(c), "r"(m));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(m), "r"(c));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(b) : "r"(m), "r"(c));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(c), "r"(m));
    asm volatile("shf.l.wrap.b32 %0, %0, %1, 31;" : "+r"(a) : "r"(b));
    asm volatile("shf.l.wrap.b32 %0, %0, %1, 31;" : "+r"(b) : "r"(a));
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a) : "r"(m), "r"(c));
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(b) : "r"(m), "r"(c));
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a) : "r"(b), "r"(c));
    asm volatile("add.u32 %0, %0, %1;" : "+r"(a) : "r"(b));
  }
  if (OP == OP_WIDE_IMAD) { /* one 64-bit multiply by a constant as mm_hash.h spells it: wide + 2 imad (+ a lop3 keeping the high word alive) */
    asm volatile("{ .reg .b32 lo, hi; mov.b64 {lo, hi}, %0; mul.wide.u32 %0, lo, %2; mov.b64 {lo, hi}, %0; lop3.b32 %1, %1, hi, %2, 0x96; }" : "+l"(w), "+r"(a) : "r"(m));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(m), "r"(c));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(b) : "r"(m), "r"(c));
  }
  if (OP == OP_HASH_ROUND) { /* half a Murmur3 body block on a dependent value, mm_hash.h's own device functions */
    uint64_t k = w ^ (uint64_t)m;
    k = mm_mulc<0x87c37b91114253d5ULL, 8>(k); k = mm_rotl<31>(k); k = mm_mulc<0x4cf5ad432745937fULL, 8>(k);
    w ^= k; w = mm_rotl<27>(w); w = mm_mul5_add<0x52dce729u>(w);
  }
  if (OP == OP_HASH19) { /* one complete 19-byte hash; the next input depends on the result */
    uint64_t ww[3] = {w, w ^ (uint64_t)c, (uint64_t)(m & 0xFFFFFFu)};
    w = mm_murmur3_k<19>(ww);
  }
}

template <int OP>
__global__ void __launch_bounds__(256) k_issue(uint32_t *out, int iters, uint32_t m0, uint32_t c0)
{
  const uint32_t m = (threadIdx.x * 2u + 1u) * m0, c = threadIdx.x ^ c0; /* per-thread register values, not constants */
  uint32_t a[CHAINS], b[CHAINS];
  uint64_t w[CHAINS];
#pragma unroll
  for (int i = 0; i < CHAINS; i++) { a[i] = threadIdx.x * 2654435761u + i; b[i] = a[i] ^ 0x9e3779b9u; w[i] = a[i]; }
  constexpr int UNR = OP == OP_HASH19 ? 2 : (OP == OP_HASH_ROUND ? 8 : UNROLL); /* keep the loop body inside the instruction cache */
  for (int it = 0; it < iters * (UNROLL / UNR); it++) {
#pragma unroll
    for (int u = 0; u < UNR; u++) {
#pragma unroll
      for (int i = 0; i < CHAINS; i++) step<OP>(a[i], b[i], w[i], m, c);
    }
  }
  uint32_t r = 0;
#pragma unroll
  for (int i = 0; i < CHAINS; i++) r ^= a[i] ^ b[i] ^ (uint32_t)w[i] ^ (uint32_t)(w[i] >> 32);
  if (r == 0x12345678u) out[blockIdx.x * blockDim.x + threadIdx.x] = r; /* keeps the chains alive */
}

template <int OP>
double run(int sm, int clock_khz, uint32_t *d_out)
{
  const int iters = 2048;
  const int grid = sm * 4, block = 256; /* 1024 threads = 32 warps per SM */
  k_issue<OP><<<grid, block>>>(d_out, 64, 3u, 5u);
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e30f;
  for (int rep = 0; rep < 5; rep++) {
    cudaEventRecord(e0);
    k_issue<OP><<<grid, block>>>(d_out, iters, 3u, 5u);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  const double warp_instr = (double)grid * (block / 32) * (double)iters * UNROLL * CHAINS * OP_INSTR[OP];
  const double clocks = best * 1e-3 * clock_khz * 1e3;
  return warp_instr / clocks / sm; /* warp instructions per clock per SM */
}

int main()
{
  cudaDeviceProp p;
  if (cudaGetDeviceProperties(&p, 0) != cudaSuccess) { fprintf(stderr, "no device\n"); return 1; }
  int clock_khz = 0;
  cudaDeviceGetAttribute(&clock_khz, cudaDevAttrClockRate, 0);
  uint32_t *d_out;
  cudaMalloc(&d_out, (size_t)p.multiProcessorCount * 4 * 256 * 4);
  double v[OP_COUNT];
  v[OP_IMAD] = run<OP_IMAD>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_IMAD_WIDE] = run<OP_IMAD_WIDE>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_SHF] = run<OP_SHF>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_LOP3] = run<OP_LOP3>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_IADD3] = run<OP_IADD3>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_PRMT] = run<OP_PRMT>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_MIX_IMAD_LOP3] = run<OP_MIX_IMAD_LOP3>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_MIX_IMAD_SHF] = run<OP_MIX_IMAD_SHF>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_MIX_WIDE_SHF] = run<OP_MIX_WIDE_SHF>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_MIX_MURMUR] = run<OP_MIX_MURMUR>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_NOWIDE_MIX] = run<OP_NOWIDE_MIX>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_WIDE_IMAD] = run<OP_WIDE_IMAD>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_HASH_ROUND] = run<OP_HASH_ROUND>(p.multiProcessorCount, clock_khz, d_out);
  v[OP_HASH19] = run<OP_HASH19>(p.multiProcessorCount, clock_khz, d_out);
  printf("{\"device\": \"%s\", \"sm_count\": %d, \"clock_mhz_nominal\": %.0f, \"unit\": \"warp instructions / clock / SM (nominal clock)\"",
         p.name, p.multiProcessorCount, clock_khz / 1e3);
  for (int i = 0; i < OP_COUNT; i++) printf(", \"%s\": %.3f", OP_NAME[i], v[i]);
  printf(", \"hash19_sass_instructions\": %d, \"hash19_per_clk_per_sm\": %.5f", (int)MM_SASS_HASH19, v[OP_HASH19] / MM_SASS_HASH19);
  printf("}\n");
  return 0;
}
