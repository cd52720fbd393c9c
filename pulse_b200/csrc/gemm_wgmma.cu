// bf16 GEMM on the Hopper tensor cores (sm_90a, wgmma): D[M,N] = epilogue(alpha * sum_k A(m,k) B(n,k)).
//
// This one kernel carries every dense contraction of the policy / value / discriminator / VAE MLPs
// (network_builder.py:105-124, amp_network_builder.py:58-249, amp_network_z_builder.py:341-467):
//   forward   Y  = act(X W^T + b)            A = X  [M,K] K-major,   B = W  [N,K] K-major
//   dgrad     dX = (dY W) * act'(.)          A = dY [M,N] K-major,   B = W  [N,K] read MN-major
//   wgrad     dW = dY^T X                    A = dY [M,N] MN-major,  B = X  [M,K] MN-major   (reduction over the batch rows)
// Operands are read as they sit in memory: the wgmma transpose bits select K-major or MN-major, nothing is transposed.
//
// Structure (persistent: one CTA per SM loops over 128 x 128 output tiles x split-K slices; 128 x 256 tiles with m64n256k16 where
// gemm_tile_n picks them):
//   warp 0       TMA producer: cp.async.bulk.tensor 2D loads (128B swizzle) into a shared-memory ring that runs continuously
//                across work items, completion on "full" mbarriers (4 stages; 6, or 5 with a pre-activation, where the epilogue is
//                register-resident: see GemmSmem);
//   warps 4..11  two consumer warpgroups, 64 rows of the tile each: wgmma.mma_async m64n128k16 (fp32 accumulators in registers),
//                one wgmma group in flight, each stage handed back to the producer ("empty") as soon as the group that read it
//                retires.  After the last k-block the same warps run the epilogue while the producer keeps filling the ring for the
//                next item:
//                  forward / input-gradient GEMMs with bf16 outputs only: straight from the accumulator registers -- bias /
//                  activation / ReLU mask words / mask-word gate -> bf16 pairs -> stmatrix into the warpgroup's shared area ->
//                  bulk tensor stores of 64 x 64 boxes;
//                  everything else: the accumulator goes to a per-warpgroup shared tile (32 x 32 fp32 blocks, 128-byte swizzle)
//                  and the epilogue runs from it: bias / activation / activation-derivative gate / column sums -> bf16 and/or fp32
//                  outputs, or bulk tensor reductions of the staged blocks into the weight-gradient buffer (split-K).
#include <cuda.h>
#include <stdlib.h>
#include <string.h>
#include <cuda_bf16.h>

#include "pulse_common.cuh"

namespace pulse {
namespace {

#ifndef PULSE_GEMM_VARIANT
#define PULSE_GEMM_VARIANT 0   // 0 = product; 3 = phase-trace build for tools/gemm_trace.py (tools/build_variant.sh trace gemm_wgmma.cu -DPULSE_GEMM_VARIANT=3)
#endif
constexpr int BM = 128, BK = 64, MMA_K = 16;
constexpr int kNarrowBN = 128, kWideBN = 256;   // output tile widths (BN, a template parameter of the kernels); see gemm_tile_n
constexpr int kConsumerWarps = 8;                 // two warpgroups
constexpr int kThreads = 128 + 32 * kConsumerWarps;   // producer warpgroup (one warp issues, three idle) + consumers
// Each consumer warp drains 32 rows x kCols columns of its warpgroup's 64 x 128 accumulator in 32-column chunks.
constexpr int kCols = 64;
constexpr int kChunks = kCols / 32;
constexpr int kStages = 4;   // ring depth of the instantiations that can take the staged epilogue, and of the wide ones
constexpr int kTmaOutF32 = 2;   // tma_out of a plain fp32 output through the register-resident epilogue (deep-ring kernels only)
constexpr unsigned kStageBytesA = BM * BK * 2;
// registers per thread of the wide kernels after setmaxnreg: the producer warpgroup gives up what the consumers' 64 x 256 fp32
// fragments (128 registers) need; 128 x (40 + 2 x 232) = 64 512 = 384 threads x 168, the launch's allocation
constexpr int kWideProducerRegs = 40, kWideConsumerRegs = 232;

// Shared memory of an instantiation with an S-stage operand ring.  The consumers hold up to two stages, so a 4-stage ring gives the
// producer two stages of lead; the update's short-K items (8-16 k-blocks) wait on operand loads for a quarter of their main loop,
// and two more stages cut the 8-k-block input-gradient items by about a quarter (DESIGN.md section 3.3).  Only the
// register-resident epilogue can afford more stages: it needs 16 KB of bf16 output boxes per consumer warpgroup
// (32 KB with the pre-activation), not the staged path's fp32 tile and per-warp tiles.  So the instantiations that may take the
// staged path keep kStages (the specialisation below), and the register-epilogue-only ones give that room to the ring: 6 stages,
// or 5 when the pre-activation boxes need the second 16 KB.
template <int S, int BN>
struct __align__(1024) GemmSmem {
  unsigned char a[S][kStageBytesA];
  unsigned char b[S][BN * BK * 2];
  unsigned char epi[2][S >= 6 ? 16384 : 32768];   // per consumer warpgroup: output boxes [0, 16 KB), pre-activation boxes [16, 32 KB);
                                                 // or one 64-column half of a plain fp32 output at a time
  float bias[2][BN];                             // per-warpgroup copy of the tile's bias
  unsigned long long full[S];
  unsigned long long empty[S];
};
template <>
struct __align__(1024) GemmSmem<kStages, kNarrowBN> {
  unsigned char a[kStages][kStageBytesA];
  unsigned char b[kStages][kNarrowBN * BK * 2];
  float epi[2][64 * kNarrowBN];            // per consumer warpgroup: 2 x 4 blocks of 32 x 32 fp32, 128-byte swizzled (4 KB each), or
                                           // (register-resident epilogue) 2 + 2 bf16 boxes of 64 x 64 for the output / pre-activation stores
  float red[kConsumerWarps][16 * 33];      // per-warp tile: bf16 store staging / fp32 transpose for atomics
  float bias[2][kNarrowBN];                // per-warpgroup copy of the tile's bias (register-resident forward epilogue)
  unsigned long long full[kStages];
  unsigned long long empty[kStages];
};
// 128 x 256 tiles (register-resident bf16 epilogue without a pre-activation): 4 stages of 16 KB A + 32 KB B (4 x 1024 clocks of
// tensor-core work in flight, as many clocks as the narrow 6-stage ring).  Each warpgroup drains its 64 x 256 fragment in two
// 128-column halves through its 16 KB area, as the narrow kernels drain their one.  No room is left for a shared bias copy: the
// wide epilogue reads the bias from global memory.
template <>
struct __align__(1024) GemmSmem<kStages, kWideBN> {
  unsigned char a[kStages][kStageBytesA];
  unsigned char b[kStages][kWideBN * BK * 2];
  unsigned char epi[2][16384];
  unsigned long long full[kStages];
  unsigned long long empty[kStages];
};
// dynamic shared memory of a launch: 1 KB of slack so the kernel can align the ring to 1024 B
template <int S, int BN>
constexpr size_t smem_bytes() { return sizeof(GemmSmem<S, BN>) + 1024; }
constexpr size_t kSmemOptin = 232448;   // sm_90 opt-in limit of dynamic shared memory per block (227 KB)
static_assert(smem_bytes<kStages, kNarrowBN>() <= kSmemOptin && smem_bytes<5, kNarrowBN>() <= kSmemOptin && smem_bytes<6, kNarrowBN>() <= kSmemOptin &&
                  smem_bytes<kStages, kWideBN>() <= kSmemOptin,
              "GEMM shared-memory layout exceeds the per-block opt-in limit");

__device__ __forceinline__ unsigned s_u32(const void* p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void g_mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(s_u32(bar)), "r"(count));
}
__device__ __forceinline__ void g_mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(s_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void g_mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(s_u32(bar)) : "memory");
}
__device__ __forceinline__ bool g_mbar_try(unsigned long long* bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(s_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void g_mbar_wait(unsigned long long* bar, unsigned parity) {
  for (int spin = 0; spin < (1 << 26); ++spin)
    if (g_mbar_try(bar, parity)) return;
  __trap();  // a protocol bug must surface as a launch error, never as a hung GPU
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, unsigned long long* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n" ::"r"(
                   s_u32(smem_dst)),
               "l"(map), "r"(s_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}
// bulk tensor store of one box from shared memory (128-byte swizzled, as the map says); completion through the bulk async-group
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, unsigned smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];\n" ::"l"(map), "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
// the same for a 3-D map ({column, row, split-K slab})
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, unsigned smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];\n" ::"l"(map), "r"(smem_src), "r"(c0), "r"(c1),
               "r"(c2)
               : "memory");
}
// four 8 x 8 bf16 matrices to shared memory; r[m] holds this thread's pair (row lane / 4, columns 2 (lane % 4) + {0, 1}) of matrix m, and
// lane l gives the 16-byte row address of row l % 8 of matrix l / 8
__device__ __forceinline__ void stmatrix_x4(unsigned addr, const unsigned (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};\n" ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3])
               : "memory");
}
__device__ __forceinline__ unsigned bf16x2_bits(__nv_bfloat162 h) { return *reinterpret_cast<unsigned*>(&h); }
// a warp's share of sum(v^2) into the fp64 accumulator: all 32 lanes call it
__device__ __forceinline__ void add_sumsq(double* sumsq, float sq) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(sumsq, static_cast<double>(sq));
}
// named barrier of one consumer warpgroup (id 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;\n" ::"r"(1 + wg) : "memory"); }

// wgmma shared-memory matrix descriptor, 128-byte swizzle: start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | SWIZZLE_128B (1) [62,64).
// K-major: rows of 64 bf16 (128 B), SBO = 1024 B between 8-row groups, LBO unused.  MN-major (the NON-reduction dimension is the
// contiguous one, e.g. dY[batch, n] read as the operand of a reduction over its rows): [64 reduction rows][64 elements] boxes of 8 KB,
// LBO = 8192 B between the 64-element MN chunks, SBO = 1024 B between 8-row reduction groups.
__device__ __forceinline__ unsigned long long gmma_desc(unsigned smem_addr, unsigned lbo) {
  unsigned long long d = 0;
  d |= static_cast<unsigned long long>((smem_addr >> 4) & 0x3fffu);
  d |= static_cast<unsigned long long>((lbo >> 4) & 0x3fffu) << 16;
  d |= static_cast<unsigned long long>(1024u >> 4) << 32;
  d |= static_cast<unsigned long long>(1u) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int NF>
__device__ __forceinline__ void acc_fence(float (&d)[NF]) {
#pragma unroll
  for (int i = 0; i < NF; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 128] (+)= A[64 x 16] B[16 x 128]; TA / TB = 1: operand is MN-major in shared memory
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], unsigned long long da, unsigned long long db, unsigned accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, "
      "%27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, "
      "%52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
      : "memory");
}
// D[64 x 256] (+)= A[64 x 16] B[16 x 256]: the wide tile's MMA (the fragment's columns 0..127 are d[0..63], 128..255 are d[64..127])
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256(float (&d)[128], unsigned long long da, unsigned long long db, unsigned accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, "
      "%27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, "
      "%52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, "
      "%77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, "
      "%101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, "
      "%121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, %131, %132;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
      : "memory");
}

__device__ __forceinline__ float act_apply(float x, int act) {
  if (act == PULSE_ACT_RELU) return fmaxf(x, 0.0f);
  if (act == PULSE_ACT_SILU) return __fdividef(x, 1.0f + __expf(-x));   // 2 MUFU ops; the IEEE division subroutine dominated the SiLU epilogue
  return x;
}
__device__ __forceinline__ float act_grad(float g, int mode) {
  // g: saved tensor -- ReLU: the layer's OUTPUT (>0 <=> active); SiLU: the layer's PRE-activation z
  if (mode == PULSE_ACT_RELU) return g > 0.0f ? 1.0f : 0.0f;
  if (mode == PULSE_ACT_SILU) {
    const float s = __fdividef(1.0f, 1.0f + __expf(-g));
    return s * (1.0f + g * (1.0f - s));
  }
  return 1.0f;
}


// Coalesced bf16 store of one epilogue warp's 32-row x 32-column block.  A lane holds 32 columns (64 bytes) of ITS row, so
// a direct 16-byte store instruction would touch 32 different rows (32 half-used sectors).  The block goes through the
// warp's private 2 KB shared tile instead (16-byte units, XOR-swizzled so both the row-wise writes and the 8-rows-at-a-time
// reads are bank-conflict free) and leaves as 8 rows x 64 contiguous bytes per instruction.  All 32 lanes must call it;
// rows >= rows_valid are not written.
__device__ __forceinline__ void store_block_bf16(uint4* st, const float (&v)[32], __nv_bfloat16* base, long long ld, int rows_valid, int lane) {
  const int sw = (lane >> 1) & 3;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = 8 * q;
    __nv_bfloat162 h0 = __floats2bfloat162_rn(v[i], v[i + 1]), h1 = __floats2bfloat162_rn(v[i + 2], v[i + 3]);
    __nv_bfloat162 h2 = __floats2bfloat162_rn(v[i + 4], v[i + 5]), h3 = __floats2bfloat162_rn(v[i + 6], v[i + 7]);
    uint4 u;
    u.x = *reinterpret_cast<unsigned*>(&h0);
    u.y = *reinterpret_cast<unsigned*>(&h1);
    u.z = *reinterpret_cast<unsigned*>(&h2);
    u.w = *reinterpret_cast<unsigned*>(&h3);
    st[lane * 4 + (q ^ sw)] = u;
  }
  __syncwarp();
  __nv_bfloat16* obase = base + (lane & 3) * 8;
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int rr = it * 8 + (lane >> 2);
    const uint4 val = st[rr * 4 + ((lane & 3) ^ ((rr >> 1) & 3))];
    if (rr < rows_valid) *reinterpret_cast<uint4*>(obase + static_cast<long long>(rr) * ld) = val;
  }
  __syncwarp();
}

#if PULSE_GEMM_VARIANT == 3   // development: per-phase clock64 trace of CTA 0 (tools/gemm_trace.py)
__device__ long long g_gemm_trace[32];
#define PULSE_TRACE(slot)                                          \
  do {                                                             \
    if (blockIdx.x == 0) g_gemm_trace[slot] = clock64();           \
  } while (0)
#define PULSE_TRACE_SET(slot, v)                                   \
  do {                                                             \
    if (blockIdx.x == 0) g_gemm_trace[slot] = (v);                 \
  } while (0)
// launch start: the slots of an earlier launch (possibly clocks of another SM) are cleared first
#define PULSE_TRACE_START()                                        \
  do {                                                             \
    if (blockIdx.x == 0) {                                         \
      for (int i_ = 1; i_ < 32; ++i_) g_gemm_trace[i_] = 0;        \
      g_gemm_trace[0] = clock64();                                 \
    }                                                              \
  } while (0)
// a ring-barrier wait that adds the clocks it spent to `clk` (stall counters of the trace)
#define PULSE_RING_WAIT(bar, parity, clk)                          \
  do {                                                             \
    const long long t_ = clock64();                                \
    g_mbar_wait(bar, parity);                                      \
    clk += clock64() - t_;                                         \
  } while (0)
#else
#define PULSE_TRACE(slot) \
  do {                    \
  } while (0)
#define PULSE_TRACE_SET(slot, v) \
  do {                           \
  } while (0)
#define PULSE_TRACE_START() \
  do {                      \
  } while (0)
#define PULSE_RING_WAIT(bar, parity, clk) g_mbar_wait(bar, parity)
#endif

// silu(z) = z / (1 + e^-z) on a bf16 pair, evaluated in fp32 (ex2.approx + rcp.approx per element) and rounded ONCE to bf16.
// A tanh.approx.bf16x2 formulation (one MUFU per two elements) has an error that is not zero-mean: at im_z_fit.yaml widths the
// encoder / prior heads came out 0.24 % small after four SiLU layers (tests/test_gpu_vae.py, full width).
__device__ __forceinline__ __nv_bfloat162 silu_bf16x2(__nv_bfloat162 z) {
  float2 f = __bfloat1622float2(z);
  f.x = __fdividef(f.x, 1.0f + __expf(-f.x));
  f.y = __fdividef(f.y, 1.0f + __expf(-f.y));
  return __floats2bfloat162_rn(f.x, f.y);
}

// Register-resident epilogue: 128 columns of the warpgroup's fp32 fragment (d[0..63], columns n0 + 8 j + 2 (lane & 3) + {0, 1}) -> bf16
// pairs -> stmatrix into the output boxes at `stage` ([0, 16 KB): two 64 x 64 boxes, 128-byte swizzle, row r = 8 16-byte units, unit u
// at u ^ (r & 7)) and, when `pre`, the rounded pre-activation into the same layout at +16 KB.  ACT runs on the rounded pair (exact for
// ReLU, which commutes with the rounding); a SiLU column group that reaches past N applies it in fp32 before the one rounding, as the
// staged epilogue does.
// stmatrix x4 at even j: matrices (j, rows r0), (j, r0 + 8), (j + 1, r0), (j + 1, r0 + 8); lane l gives the address of row l % 8 of
// matrix l / 8.
template <int ACT>
__device__ __forceinline__ void stage_tile_bf16(const float* d, unsigned stage, bool pre, int n0, int N) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned srow = stage + ((warp & 3) * 16 + ((lane >> 3) & 1) * 8 + (lane & 7)) * 128;
  const int sj = lane >> 4;
  const __nv_bfloat162 zero2 = __float2bfloat162_rn(0.0f);
#pragma unroll
  for (int j = 0; j < kNarrowBN / 8; j += 2) {
    const bool full_half = n0 + 64 * (j >> 3) + 64 <= N;
    unsigned o[4], p[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = 4 * (j + (k >> 1)) + 2 * (k & 1);
      __nv_bfloat162 h = __floats2bfloat162_rn(d[i], d[i + 1]);
      p[k] = bf16x2_bits(h);
      if (ACT == PULSE_ACT_RELU) h = __hmax2(h, zero2);
      if (ACT == PULSE_ACT_SILU) h = full_half ? silu_bf16x2(h) : __floats2bfloat162_rn(act_apply(d[i], ACT), act_apply(d[i + 1], ACT));
      o[k] = bf16x2_bits(h);
    }
    const unsigned addr = srow + (j >> 3) * 8192 + ((((j & 7) + sj) ^ (lane & 7)) << 4);
    stmatrix_x4(addr, o);
    if (pre) stmatrix_x4(addr + 16384, p);
  }
}

// A_MN / B_MN: operand is MN-major in global memory ([reduction rows, non-reduction cols] row-major) instead of K-major.
// MODE selects which epilogue features are COMPILED IN: the fully general epilogue is several thousand SASS instructions per
// instance, so each specialisation carries only what its caller can ask for (instruction-cache footprint); the host picks the
// smallest one that covers the request.
enum : int { kModeGeneric = 0, kModeFwd = 1, kModeDgrad = 2, kModeWgrad = 3, kModeDgradVec = 4 };

#include "gemm_kernel.inc"

// ---- host side: tensor maps through the driver entry point (no link-time libcuda dependency) ------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// rows x cols bf16 matrix, row stride ld elements, box `box_rows` rows x 64 cols, 128B swizzle, OOB reads return 0.
// K-major operand: rows = M (or N), cols = K, box 128 x 64.  MN-major operand: rows = K (reduction), cols = M (or N), box 64 x 64.
bool make_map(CUtensorMap* map, const void* base, long long rows, long long cols, long long ld, unsigned box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return false;
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {BK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// fp32 [rows, cols] output (row stride ld floats) as a tensor map with 32 x 32 boxes, 128-byte swizzle: the target of the weight-gradient
// epilogue's bulk tensor reductions (out-of-range rows / columns of a box are clipped by the hardware).
bool make_map_c(CUtensorMap* map, const float* base, long long rows, long long cols, long long ld) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return false;
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 4};
  cuuint32_t box[2] = {32, 32};
  cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// fp32 split-K slabs [splits][rows, cols] (slab z at base + z * split_stride floats, row stride ld floats) as a 3-D tensor map with 32 x 32 x 1
// boxes, 128-byte swizzle: the target of the register-resident epilogue's fp32 stores (rows / columns beyond the slab are clipped).
bool make_map_slabs(CUtensorMap* map, const float* base, long long splits, long long rows, long long cols, long long ld, long long split_stride) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return false;
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(splits)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(ld) * 4, static_cast<cuuint64_t>(splits > 1 ? split_stride : rows * ld) * 4};
  cuuint32_t box[3] = {32, 32, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// the reduction path needs 16-byte aligned rows and N a multiple of 4: the bulk tensor reduction clips the column tail in whole
// 16-byte units, so at N = 69 it would add (zeros) into columns 69..71, outside the output.  Otherwise the kernel uses fp32 atomics.
bool tma_reduce_ok(const pulse_gemm_epilogue_t& ep, long long n) {
  return ep.out_f32 != nullptr && ep.accumulate && (n % 4) == 0 && (ep.ldf % 4) == 0 && (reinterpret_cast<uintptr_t>(ep.out_f32) % 16) == 0;
}
bool tma_rows_ok(const void* base, long long ld) { return (ld % 8) == 0 && (reinterpret_cast<uintptr_t>(base) % 16) == 0; }

// Tensor maps of the epilogue and whether the kernel uses them (tma_out):
//   wgrad: map_c = the fp32 gradient, target of the bulk tensor reductions;
//   forward / input gradient with bf16 outputs only (no fp32 or transposed copy, bf16 gate or column sums): the register-resident
//   epilogue, map_c = out, map_p = preact, [M, N] bf16 with 64 x 64 boxes, so the hardware clips the row and column tails.  It clips
//   columns in whole 16-byte units, so N must be a multiple of 8 (an N = 69 store would overwrite columns 69..71).
//   forward with a plain fp32 output only (split-K slabs of the weight gradients: no alpha, bias, activation or other output), N a
//   multiple of 4: the register-resident epilogue of the deep-ring kernel, map_c = the slabs (tma_out = kTmaOutF32).  The 4-stage kernel
//   has no such path: the launch clears tma_out when it runs that one.
// Anything else, or rows that are not 16-byte aligned, runs the staged epilogue.
int epilogue_maps(int mode, const pulse_gemm_epilogue_t& ep, long long m, long long n, int splits, CUtensorMap* map_c, CUtensorMap* map_p,
                  int* tma_out) {
  memset(map_c, 0, sizeof(*map_c));
  memset(map_p, 0, sizeof(*map_p));
  *tma_out = 0;
  if (mode == kModeWgrad) {
    if (!tma_reduce_ok(ep, n)) return PULSE_OK;
    if (!make_map_c(map_c, ep.out_f32, m, n, ep.ldf)) {
      set_error("pulse_gemm_bf16: cuTensorMapEncodeTiled failed for the fp32 output");
      return PULSE_ERR_CUDA;
    }
    *tma_out = 1;
    return PULSE_OK;
  }
  if (mode == kModeFwd && ep.out_f32 != nullptr && ep.out == nullptr && ep.out_t == nullptr && ep.preact == nullptr && ep.relu_mask == nullptr &&
      ep.bias == nullptr && ep.act == PULSE_ACT_NONE && ep.alpha == 1.0f && !ep.accumulate && (n % 4) == 0 && (ep.ldf % 4) == 0 &&
      (reinterpret_cast<uintptr_t>(ep.out_f32) % 16) == 0 && (splits == 1 || (ep.split_stride % 4) == 0)) {
    if (!make_map_slabs(map_c, ep.out_f32, splits, m, n, ep.ldf, ep.split_stride)) {
      set_error("pulse_gemm_bf16: cuTensorMapEncodeTiled failed for the fp32 output");
      return PULSE_ERR_CUDA;
    }
    *tma_out = kTmaOutF32;
    return PULSE_OK;
  }
  if ((mode != kModeFwd && mode != kModeDgrad) || (n % 8) != 0 || ep.out == nullptr || ep.out_f32 != nullptr || ep.out_t != nullptr || ep.gate != nullptr ||
      ep.colsum != nullptr || !tma_rows_ok(ep.out, ep.ldo) || (ep.preact != nullptr && !tma_rows_ok(ep.preact, ep.ldp)))
    return PULSE_OK;
  if (!make_map(map_c, ep.out, m, n, ep.ldo, 64) || (ep.preact != nullptr && !make_map(map_p, ep.preact, m, n, ep.ldp, 64))) {
    set_error("pulse_gemm_bf16: cuTensorMapEncodeTiled failed for the bf16 output");
    return PULSE_ERR_CUDA;
  }
  *tma_out = 1;
  return PULSE_OK;
}

int gemm_num_sms() {
  static int limited = 0;
  if (limited == 0) {
    int dev = 0, num_sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    // PULSE_GEMM_SMS=n: leave SMs free for a concurrent collective (the persistent grid otherwise owns the whole GPU)
    limited = num_sms;
    const char* e = getenv("PULSE_GEMM_SMS");
    if (e != nullptr && atoi(e) >= 1 && atoi(e) < num_sms) limited = atoi(e);
  }
  return limited;
}

// Ring depth of a launch whose epilogue is register-resident (reg_epi) or not: see GemmSmem.  PULSE_GEMM_STAGES=4 keeps every launch
// on the 4-stage kernel; it is read at every launch, so one process can compare both kernels.
int ring_stages(bool reg_epi, bool preact) {
  const char* e = getenv("PULSE_GEMM_STAGES");
  const bool force4 = e != nullptr && atoi(e) == kStages;
  return (!reg_epi || force4) ? kStages : preact ? 5 : 6;
}

// Output tile width of an m x n GEMM whose work items run kb_per_item k-blocks, split-K `splits`, on `sms` persistent CTAs.  A
// 128 x 256 k-block moves 48 KB into shared memory for 1024 tensor-core clocks, a quarter fewer bytes per MMA clock than the 32 KB /
// 512 clocks of a 128 x 128 one, and the narrow main loops are bound by that operand stream (DESIGN.md section 3.3).  The wide tile is
// taken where it does not cost a round: twice the work per item, so 2 x its rounds must not exceed the narrow rounds (an M = 12288,
// N = 512 GEMM has 192 wide items, 2 rounds, against 384 narrow ones, 3 rounds).  Items of fewer than kWideMinKb k-blocks are mostly
// epilogue and ring fill, which the wide tile does not shorten.
constexpr int kWideMinKb = 4;
int gemm_tile_n(long long m, long long n, int kb_per_item, int splits, int sms) {
  if (n < kWideBN || kb_per_item < kWideMinKb || sms < 1) return kNarrowBN;
  const long long tm = (m + BM - 1) / BM;
  const long long rounds_narrow = (tm * ((n + kNarrowBN - 1) / kNarrowBN) * splits + sms - 1) / sms;
  const long long rounds_wide = (tm * ((n + kWideBN - 1) / kWideBN) * splits + sms - 1) / sms;
  return 2 * rounds_wide <= rounds_narrow ? kWideBN : kNarrowBN;
}

// PULSE_GEMM_BN=128 keeps every launch on the 128 x 128 tile (to compare both widths in one process; read at every launch).  The
// default is always the shape rule above.
bool narrow_forced() {
  const char* e = getenv("PULSE_GEMM_BN");
  return e != nullptr && atoi(e) == kNarrowBN;
}
// the last GEMM launch issued from the host (pulse_gemm_last_launch): mode, ring depth, tile width, tma_out, splits, grid
int g_last_launch[6] = {};

// sets the kernel's dynamic shared-memory size once per instantiation and checks it against the device's opt-in limit
template <typename Kernel>
int set_smem_once(Kernel kernel, size_t bytes, bool* done) {
  if (*done) return PULSE_OK;
  int dev = 0, optin = 0;
  PULSE_CUDA_OK(cudaGetDevice(&dev));
  PULSE_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  PULSE_REQUIRE(bytes <= static_cast<size_t>(optin), "pulse_gemm_bf16: the GEMM needs %zu bytes of shared memory per block, the device allows %d",
                bytes, optin);
  PULSE_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes)));
  *done = true;
  return PULSE_OK;
}

template <bool A_MN, bool B_MN, int MODE, int S, int BN>
int launch_gemm_ring(const CUtensorMap& map_a, const CUtensorMap& map_b, const CUtensorMap& map_c, const CUtensorMap& map_p,
                     const pulse_gemm_epilogue_t& ep, int m, int n, int k, int splits, int kb_per_split, int tma_out, cudaStream_t stream) {
  static bool attr_set = false;
  const int rc = set_smem_once(gemm_bf16_kernel<A_MN, B_MN, MODE, S, BN>, smem_bytes<S, BN>(), &attr_set);
  if (rc != PULSE_OK) return rc;
  const int num_sms = gemm_num_sms();
  PULSE_REQUIRE(num_sms > 0, "pulse_gemm_bf16: cannot query the device's SM count");
  // persistent: one CTA per SM loops over the work items
  const long long total = static_cast<long long>((n + BN - 1) / BN) * ((m + BM - 1) / BM) * splits;
  const unsigned grid = static_cast<unsigned>(total < num_sms ? total : num_sms);
  static int use_pdl = -1;
  if (use_pdl < 0) {
    const char* e = getenv("PULSE_GEMM_PDL");
    use_pdl = (e != nullptr && e[0] == '0') ? 0 : 1;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid, 1, 1);
  cfg.blockDim = dim3(kThreads, 1, 1);
  cfg.dynamicSmemBytes = smem_bytes<S, BN>();
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (use_pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  PULSE_CUDA_OK(cudaLaunchKernelEx(&cfg, gemm_bf16_kernel<A_MN, B_MN, MODE, S, BN>, map_a, map_b, map_c, map_p, ep, m, n, k, kb_per_split, splits, tma_out));
  PULSE_LAUNCH_OK("gemm_bf16_kernel");
  const int launch[6] = {MODE, S, BN, tma_out, splits, static_cast<int>(grid)};
  memcpy(g_last_launch, launch, sizeof(launch));
  return PULSE_OK;
}

// b / ldb: the B operand, for the wide tile's map (a K-major B box spans the tile's BN rows)
template <bool A_MN, bool B_MN, int MODE>
int launch_gemm(const CUtensorMap& map_a, const CUtensorMap& map_b, const void* b, long long ldb, const pulse_gemm_epilogue_t& ep, int m, int n,
                int k, int splits, int kb_per_split, cudaStream_t stream) {
  CUtensorMap map_c, map_p;
  int tma_out = 0;
  const int rc = epilogue_maps(MODE, ep, m, n, splits, &map_c, &map_p, &tma_out);
  if (rc != PULSE_OK) return rc;
  if constexpr (MODE == kModeFwd || MODE == kModeDgrad) {
    const int s = ring_stages(tma_out != 0, ep.preact != nullptr);
    if (s == kStages && tma_out == kTmaOutF32) tma_out = 0;
    if constexpr (!A_MN) {   // A MN-major is a weight gradient: those keep the narrow tile
      // wide: the bf16 register-resident epilogue without a pre-activation (the 16 KB areas hold no pre-activation boxes)
      if (s != kStages && tma_out == 1 && ep.preact == nullptr && !narrow_forced() &&
          gemm_tile_n(m, n, kb_per_split, splits, gemm_num_sms()) == kWideBN) {
        CUtensorMap map_bw = map_b;
        if (!B_MN && !make_map(&map_bw, b, n, k, ldb, kWideBN)) {
          set_error("pulse_gemm_bf16: cuTensorMapEncodeTiled failed for the wide B operand");
          return PULSE_ERR_CUDA;
        }
        return launch_gemm_ring<A_MN, B_MN, MODE, kStages, kWideBN>(map_a, map_bw, map_c, map_p, ep, m, n, k, splits, kb_per_split, tma_out, stream);
      }
    }
    if (s == 6) return launch_gemm_ring<A_MN, B_MN, MODE, 6, kNarrowBN>(map_a, map_b, map_c, map_p, ep, m, n, k, splits, kb_per_split, tma_out, stream);
    if constexpr (MODE == kModeFwd) {   // only the forward epilogue writes a pre-activation
      if (s == 5) return launch_gemm_ring<A_MN, B_MN, MODE, 5, kNarrowBN>(map_a, map_b, map_c, map_p, ep, m, n, k, splits, kb_per_split, tma_out, stream);
    }
  }
  return launch_gemm_ring<A_MN, B_MN, MODE, kStages, kNarrowBN>(map_a, map_b, map_c, map_p, ep, m, n, k, splits, kb_per_split, tma_out, stream);
}

int epilogue_mode(const pulse_gemm_epilogue_t* ep) {
  const bool want_fwd = ep->bias || ep->act != PULSE_ACT_NONE || ep->preact || ep->out_t || ep->relu_mask;
  const bool want_dgrad = ep->gate || ep->colsum || ep->sumsq || ep->gate_mask;
  const bool want_accum = ep->accumulate != 0;
  if (!want_dgrad && !want_accum) return kModeFwd;
  if (!want_fwd && !want_accum) return (ep->gate && ep->gate_mode != PULSE_ACT_RELU) ? kModeDgradVec : kModeDgrad;
  // the weight-gradient epilogue adds the raw accumulator (bulk reductions of the staged tile, or atomics): no alpha
  if (!want_fwd && !want_dgrad && !ep->out && ep->alpha == 1.0f) return kModeWgrad;
  return kModeGeneric;
}

}  // namespace
}  // namespace pulse

#if PULSE_GEMM_VARIANT == 3
extern "C" int pulse_debug_gemm_trace(long long* out) {
  return cudaMemcpyFromSymbol(out, pulse::g_gemm_trace, sizeof(long long) * 32) == cudaSuccess ? 0 : -2;
}
#endif

extern "C" int pulse_gemm_num_splits(int64_t k, int32_t split_k) {
  const int num_kb = static_cast<int>((k + 63) / 64);
  int splits = split_k < 1 ? 1 : (split_k > num_kb ? num_kb : split_k);
  const int kb_per_split = (num_kb + splits - 1) / splits;
  return (num_kb + kb_per_split - 1) / kb_per_split;  // every slab gets at least one k-block
}

// the shape rule alone (gemm_tile_n): the width it picks for an m x n x k GEMM with split_k on `sms` SMs.  A launch takes it only where a
// wide instantiation applies (see launch_gemm); pulse_gemm_last_launch reports what a launch took.
extern "C" int pulse_gemm_tile_n(int64_t m, int64_t n, int64_t k, int32_t split_k, int32_t sms) {
  const int num_kb = static_cast<int>((k + 63) / 64);
  const int splits = pulse_gemm_num_splits(k, split_k);
  return pulse::gemm_tile_n(m, n, (num_kb + splits - 1) / splits, splits, sms);
}

// the kernel the last GEMM launch issued from the host took: {epilogue mode, ring depth, tile width, tma_out, splits, grid}; zeros
// before the first
extern "C" int pulse_gemm_last_launch(int32_t* out) {
  using namespace pulse;
  PULSE_REQUIRE(out != nullptr, "pulse_gemm_last_launch: null argument");
  memcpy(out, pulse::g_last_launch, sizeof(pulse::g_last_launch));
  return PULSE_OK;
}

// output tile width (128 or 256) of the last GEMM launch issued from the host; 0 before the first (field 2 of pulse_gemm_last_launch)
extern "C" int pulse_gemm_last_tile_n(void) { return pulse::g_last_launch[2]; }

// flags: bit 0 = A is MN-major ([K, M] row-major in memory), bit 1 = B is MN-major ([K, N] row-major in memory)
extern "C" int pulse_gemm_bf16(const void* a, int64_t lda, const void* b, int64_t ldb, int64_t m, int64_t n, int64_t k,
                               const pulse_gemm_epilogue_t* ep, int32_t split_k, uint32_t flags, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(a && b && ep, "pulse_gemm_bf16: null argument");
  PULSE_REQUIRE(m > 0 && n > 0 && k > 0, "pulse_gemm_bf16: empty problem %lld x %lld x %lld", (long long)m, (long long)n, (long long)k);
  PULSE_REQUIRE(m < (1ll << 31) && n < (1ll << 31) && k < (1ll << 31), "pulse_gemm_bf16: dimension too large");
  PULSE_REQUIRE((flags & ~3u) == 0, "pulse_gemm_bf16: bad flags");
  const bool a_mn = flags & PULSE_GEMM_A_MN, b_mn = flags & PULSE_GEMM_B_MN;
  PULSE_REQUIRE(lda >= (a_mn ? m : k) && ldb >= (b_mn ? n : k) && (lda % 8) == 0 && (ldb % 8) == 0,
                "pulse_gemm_bf16: leading dimensions must cover the contiguous extent and be multiples of 8 (16-byte rows), got %lld %lld",
                (long long)lda, (long long)ldb);
  PULSE_REQUIRE(aligned16(a) && aligned16(b), "pulse_gemm_bf16: operands must be 16-byte aligned");
  PULSE_REQUIRE(ep->out || ep->out_t || ep->out_f32, "pulse_gemm_bf16: no output requested");
  PULSE_REQUIRE(split_k >= 1, "pulse_gemm_bf16: split_k must be >= 1");
  PULSE_REQUIRE(split_k == 1 || (ep->out_f32 && !ep->out && !ep->out_t && !ep->bias && ep->act == PULSE_ACT_NONE && !ep->gate && !ep->preact && !ep->colsum),
                "pulse_gemm_bf16: split-K only supports plain fp32 outputs (slabs or atomic accumulation)");
  PULSE_REQUIRE(ep->gate == nullptr || ep->gate_mode == PULSE_ACT_RELU || ep->gate_mode == PULSE_ACT_SILU, "pulse_gemm_bf16: bad gate_mode");
  PULSE_REQUIRE((ep->relu_mask == nullptr || ep->ld_rmask >= m) && (ep->gate_mask == nullptr || ep->ld_gmask >= m),
                "pulse_gemm_bf16: mask word rows must hold at least M entries");
  PULSE_REQUIRE(!(ep->gate_mask && ep->gate), "pulse_gemm_bf16: give the ReLU gate either as bf16 activations or as bit words, not both");
  CUtensorMap map_a, map_b;
  const bool ok_a = a_mn ? make_map(&map_a, a, k, m, lda, 64) : make_map(&map_a, a, m, k, lda, BM);
  const bool ok_b = b_mn ? make_map(&map_b, b, k, n, ldb, 64) : make_map(&map_b, b, n, k, ldb, kNarrowBN);
  if (!ok_a || !ok_b) {
    set_error("pulse_gemm_bf16: cuTensorMapEncodeTiled failed (driver entry point missing or bad strides)");
    return PULSE_ERR_CUDA;
  }
  const int num_kb = static_cast<int>((k + BK - 1) / BK);
  const int splits = pulse_gemm_num_splits(k, split_k);
  const int kb_per_split = (num_kb + splits - 1) / splits;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // smallest epilogue specialisation that covers the request (see the MODE comment on the kernel)
  const int mode = epilogue_mode(ep);
  const int mi = (int)m, ni = (int)n, ki = (int)k;
#define PULSE_GEMM_DISPATCH(AM, BM_)                                                                                                 \
  switch (mode) {                                                                                                                    \
    case kModeFwd: return launch_gemm<AM, BM_, kModeFwd>(map_a, map_b, b, ldb, *ep, mi, ni, ki, splits, kb_per_split, st);           \
    case kModeDgrad: return launch_gemm<AM, BM_, kModeDgrad>(map_a, map_b, b, ldb, *ep, mi, ni, ki, splits, kb_per_split, st);       \
    case kModeWgrad: return launch_gemm<AM, BM_, kModeWgrad>(map_a, map_b, b, ldb, *ep, mi, ni, ki, splits, kb_per_split, st);       \
    case kModeDgradVec: return launch_gemm<AM, BM_, kModeDgradVec>(map_a, map_b, b, ldb, *ep, mi, ni, ki, splits, kb_per_split, st); \
    default: return launch_gemm<AM, BM_, kModeGeneric>(map_a, map_b, b, ldb, *ep, mi, ni, ki, splits, kb_per_split, st);             \
  }
  if (a_mn && b_mn) { PULSE_GEMM_DISPATCH(true, true) }
  if (a_mn) { PULSE_GEMM_DISPATCH(true, false) }
  if (b_mn) { PULSE_GEMM_DISPATCH(false, true) }
  PULSE_GEMM_DISPATCH(false, false)
#undef PULSE_GEMM_DISPATCH
}
