// Device primitives for sm_90a (Hopper): mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA with operands in
// shared memory or, for A, in registers) and its shared-memory descriptors, and the small math, warp-reduction and gpu-scope
// hand-off helpers the kernel files share.  Inline PTX only - no CUTLASS dependency.
//
// Conventions used by every kernel in this library:
//   * GEMM operands are "split-bf16": a 32-bit value v is stored as two bf16 planes hi = bf16(v), lo = bf16(v - hi)
//     (16-bit effective mantissa).  A product A*B is evaluated as A_hi*B_hi + A_lo*B_hi + A_hi*B_lo with fp32
//     accumulation in registers (3 wgmma per K-step) - relative error ~2^-16, which keeps the fp32 1e-3 parity
//     contract through 30 residual layers where a single TF32 pass does not (measured in DESIGN.md).
//   * Operand tiles are K-major, 64 bf16 (=128 B) per row, 128B-swizzled, written by TMA and read by wgmma.
//   * Accumulator fragments (wgmma m64nN, f32): warp w of the warpgroup owns rows 16 w + g and 16 w + g + 8 (g = lane / 4);
//     d[4 j + {0, 1}] are row 16 w + g, columns 8 j + 2 (lane % 4) + {0, 1}; d[4 j + {2, 3}] the same columns of row + 8.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pk {

constexpr int kSwizzleBytes = 128;     // one K-chunk row: 64 bf16
constexpr int kChunkK = 64;            // bf16 elements per K-chunk

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------------------------
// proxies / fences
// ----------------------------------------------------------------------------------------------------------------
// all generic-proxy writes of this thread -> visible to later async-proxy (TMA / wgmma) reads
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
// the same for this thread's shared-memory writes only (e.g. a tile staged for a TMA store); global writes are not waited for
__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}

// ----------------------------------------------------------------------------------------------------------------
// wgmma
// ----------------------------------------------------------------------------------------------------------------
constexpr int kWgmmaK = 16;            // K per wgmma.mma_async (bf16)

// Shared-memory matrix descriptor: K-major tile, rows of 128 B, SWIZZLE_128B, 8-row groups 1024 B apart; the tile must be
// 1024-B aligned (base offset 0).  Advancing the start address by 32 B selects the next K-step of 16 inside the 128 B row.
// (bit layout: start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | base offset [49,52) | layout 1 = SWIZZLE_128B [62,64))
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;             // LBO (unused for swizzled K-major; canonical value 1)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;     // SBO: 8 rows * 128 B
  d |= static_cast<uint64_t>(1) << 62;             // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ uint64_t desc_kstep(int k) { return static_cast<uint64_t>((k * kWgmmaK * 2) >> 4); }
// The same for a tile of ONE K-step: rows of 32 B (16 bf16), SWIZZLE_32B, 8-row groups 256 B apart, 256-B aligned.
__device__ __forceinline__ uint64_t make_smem_desc_sw32(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;             // LBO (unused: the K extent is one swizzle atom)
  d |= static_cast<uint64_t>(256 >> 4) << 32;      // SBO: 8 rows * 32 B
  d |= static_cast<uint64_t>(3) << 62;             // SWIZZLE_32B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// register budget of the executing warpgroup (all of its warps execute it): producers give registers back, consumers take them
template <uint32_t kRegs>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <uint32_t kRegs>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
// named barrier over `threads` threads (a warpgroup: 128)
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// arrive without waiting: the other `threads` - 128 threads of the barrier wait on it with named_bar_sync
__device__ __forceinline__ void named_bar_arrive(int id, int threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// wgmma.mma_async m64nNk16, bf16 x bf16 -> f32, K-major operands; d (N / 2 floats per thread) is accumulated in place.
// ss: A and B from shared memory (descriptors); rs: A from registers (the m64k16 A fragment, 4 x bf16x2 per thread).
#define PK_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define PK_F32(i) PK_F8(i), PK_F8(i + 8), PK_F8(i + 16), PK_F8(i + 24)
#define PK_D32 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
#define PK_D64 PK_D32 ",%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
#define PK_D96 PK_D64 ",%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95"
#define PK_D128 PK_D96 ",%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {" PK_D32 "}, %32, %33, p, 1, 1, 0, 0;\n}\n"
               : PK_F32(0) : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {" PK_D64 "}, %64, %65, p, 1, 1, 0, 0;\n}\n"
               : PK_F32(0), PK_F32(32) : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_ss_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {" PK_D128 "}, %128, %129, p, 1, 1, 0, 0;\n}\n"
               : PK_F32(0), PK_F32(32), PK_F32(64), PK_F32(96) : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {" PK_D32 "}, {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n}\n"
               : PK_F32(0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {" PK_D64 "}, {%64,%65,%66,%67}, %68, p, 1, 1, 0;\n}\n"
               : PK_F32(0), PK_F32(32) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_rs_n192(float (&d)[96], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %101, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 {" PK_D96 "}, {%96,%97,%98,%99}, %100, p, 1, 1, 0;\n}\n"
               : PK_F32(0), PK_F32(32), PK_F32(64) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
#undef PK_F32
#undef PK_F8

// ----------------------------------------------------------------------------------------------------------------
// split-bf16 helpers
// ----------------------------------------------------------------------------------------------------------------
// Philox4x32-10 (counter c0..c3, key k0, k1): the dropout generator of pk_dropout (train.cu) and of the Tacotron2 prenet
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t* out) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// element i of a split-bf16 tensor as fp32
__device__ __forceinline__ float ld_split(const __nv_bfloat16* hi, const __nv_bfloat16* lo, long long i) {
  return __bfloat162float(hi[i]) + __bfloat162float(lo[i]);
}
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}
__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return static_cast<uint32_t>(__bfloat16_as_ushort(a)) | (static_cast<uint32_t>(__bfloat16_as_ushort(b)) << 16);
}
// split 8 floats -> two uint4 of packed bf16 (hi plane, lo plane)
__device__ __forceinline__ void split8(const float* v, uint4& hi, uint4& lo) {
  __nv_bfloat16 h[8], l[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) split_bf16(v[i], h[i], l[i]);
  hi = make_uint4(pack_bf16x2(h[0], h[1]), pack_bf16x2(h[2], h[3]), pack_bf16x2(h[4], h[5]), pack_bf16x2(h[6], h[7]));
  lo = make_uint4(pack_bf16x2(l[0], l[1]), pack_bf16x2(l[2], l[3]), pack_bf16x2(l[4], l[5]), pack_bf16x2(l[6], l[7]));
}
// split two fp32 values into packed bf16x2 hi / lo words (cvt.rn.bf16x2.f32: one instruction per pair)
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  const float ra = a - __uint_as_float(hi << 16);
  const float rb = b - __uint_as_float(hi & 0xffff0000u);
  const __nv_bfloat162 l = __floats2bfloat162_rn(ra, rb);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// ----------------------------------------------------------------------------------------------------------------
// math, warp reductions, gpu-scope hand-offs
// ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2_approx(float x) {   // MUFU.EX2, 2 ulp; inf for x > 128, 0 for x < -150
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {   // MUFU.RCP, 1 ulp; rcp(inf) = 0
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// Sum of v over a block of kThreads threads (a power of two) as a fixed-order tree in double; red holds kThreads doubles.
// Every thread returns the sum, and red may be reused right away.
template <int kThreads>
__device__ __forceinline__ double block_sum_tree(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}
// for (i = global thread index; i < n; i += all threads of the grid): launch with grid_stride_blocks (pk_host.h)
#define PK_GRID_STRIDE(i, n) \
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < (n); i += static_cast<long long>(gridDim.x) * blockDim.x)
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_inc(unsigned* p) {
  asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p) : "memory");
}


// ----------------------------------------------------------------------------------------------------------------
// Shared-memory access by 32-bit shared-space address.  Kernels round their dynamic smem base up to 1024 B with
// integer arithmetic, after which the compiler can no longer prove a pointer is in shared space and would emit
// generic LD/ST (long-scoreboard latency); these helpers keep the accesses on the LDS/STS path.
// ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 lds_f4(uint32_t addr) {   // ordered w.r.t. the other volatile smem helpers
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ float2 lds_f2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void sts_f2(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

// mbarrier / TMA helpers taking shared-space addresses
__device__ __forceinline__ void mbar_init_a(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx_a(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive_a(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Bounded spin: a protocol bug must trap (-> launch error reported through the C-ABI), never hang the GPU.
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  for (uint32_t spin = 0; spin < (1u << 26); ++spin) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) return;
  }
  __trap();
}
__device__ __forceinline__ void tma_load_3d_a(uint32_t smem_dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d_a(uint32_t smem_dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// TMA store of a box (rows outside the tensor are not written); the smem source may be reused after bulk_wait_read<0>.
// The generic-proxy writes that filled the source must be made visible first (fence_proxy_async_all + a barrier).
__device__ __forceinline__ void tma_store_4d_a(const CUtensorMap* tm, uint32_t smem_src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d_a(const CUtensorMap* tm, uint32_t smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
// The same, adding the box element-wise onto global memory (the add happens in L2; rows outside the tensor are left alone).
__device__ __forceinline__ void tma_reduce_add_3d_a(const CUtensorMap* tm, uint32_t smem_src, int c0, int c1, int c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }


// ----------------------------------------------------------------------------------------------------------------
// Accumulator staging: a warpgroup's m64 x 32-column slice of a wgmma accumulator goes through a [64][32] fp32 slot of
// shared memory (8 KB, 16-byte chunks XOR-swizzled by row) so that a thread can then read one whole row of it - the
// row-per-thread layout the epilogues are written in.
// ----------------------------------------------------------------------------------------------------------------
constexpr int kStageSlotBytes = 64 * 32 * 4;
__device__ __forceinline__ uint32_t stage_addr(uint32_t slot, int row, int col) {   // col: multiple of 2
  return slot + row * 128 + ((((col >> 2) ^ (row & 7)) << 4) | ((col & 3) << 2));
}
// columns [32 C, 32 C + 32) of the accumulator d; wg_thread = thread index inside the warpgroup.  Call it from fully
// unrolled loops only: C must fold to a constant, or the accumulator would be indexed dynamically (local memory).
template <int R>
__device__ __forceinline__ void stage_store(uint32_t slot, const float (&d)[R], int C, int wg_thread) {
  const int w = wg_thread >> 5, lane = wg_thread & 31;
  const int r0 = 16 * w + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = 4 * C + jj;
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stage_addr(slot, r0, 8 * jj + c0)), "f"(d[4 * j]), "f"(d[4 * j + 1]) : "memory");
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stage_addr(slot, r0 + 8, 8 * jj + c0)), "f"(d[4 * j + 2]), "f"(d[4 * j + 3])
                 : "memory");
  }
}
__device__ __forceinline__ void stage_load_row(uint32_t slot, int row, float (&v)[32]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float4 x = lds_f4(slot + row * 128 + ((k ^ (row & 7)) << 4));
    v[4 * k] = x.x; v[4 * k + 1] = x.y; v[4 * k + 2] = x.z; v[4 * k + 3] = x.w;
  }
}

}  // namespace pk
