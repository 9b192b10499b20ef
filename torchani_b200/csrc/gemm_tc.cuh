// Persistent, warp-specialised, TMA-fed wgmma grouped GEMM for the ensemble MLP (sm_90a).
//
//   C[128-row tile, bn] = epilogue( A[128, K] x B[bn, K]^T )        both operands K-major
//
// fp32 accuracy on the tensor cores from 16-bit pieces (common.cuh, ANI_OPND_FP16X2):
//   * default "2 x fp16": every fp32 operand x is stored as two IEEE half pieces of s*x
//     (s*x = p1 + p2, residual < 2^-22 |s*x|; s = a power of two per operand class that keeps p2 a
//     normal half); every K-step issues three products,
//         a2 b1, a1 b2, a1 b1          (the dropped a2 b2 is < 2^-22 relative),
//     into one fp32 accumulator; the epilogue multiplies by 1/(s_a s_b) (exact).
//   * "3 x bf16": x = p1 + p2 + p3 bfloat16 pieces, six products (a3b1, a1b3, a2b2, a2b1, a1b2,
//     a1b1), 6 bytes per element, no scale.
//
// BOTH operands live in global memory in the "tiled operand" layout of include/ani_b200.h:
// 32-column K-blocks, [p1 rows x 64 B | p2 rows x 64 B (| p3 rows x 64 B)], every 8-row group in
// SWIZZLE_64B order -- the layout wgmma's 64-byte-swizzled K-major shared-memory descriptors read.
// A K-block of a tile is therefore ONE contiguous byte range that one thread moves with
// cp.async.bulk (TMA) straight into shared memory; no thread ever touches operand data on the way in.
//
// Roles (3 warpgroups, one CTA per SM, persistent over a device-side list of work units):
//   warp  0     producer: one lane arms the mbarrier (expect_tx) and issues the bulk copies (warps 1-3 only
//               hand their registers over to the consumers and exit)
//   warps 4-11  two consumer warpgroups: warpgroup w owns rows 64w .. 64w+63 of the tile, issues
//               wgmma.m64n64k16 per 64-column slice from the shared-memory ring into a
//               register accumulator of up to 64 x 256, then runs the epilogue straight from registers:
//               bias + CELU | * CELU'(stored activation) | final layer + gradient seed | plain
//               (GELU models, ACT_GELU: GELU without bias, storing GELU' beside the activation | * stored GELU' |
//               GELU head)
// Ring: STAGES slots of (A block + B block of up to 256 rows); the producer runs ahead across units, so
// the loads of the next unit overlap the epilogue of the current one.
//
// Work lists (StepArgs): ONE phase (a plain GEMM launch, chained in stream order), or the whole MLP of a
// step (3 or 6 phases) in one launch.  Layer k of (row tile r, member m) needs only layer k-1 of (r, m), so
// units are ordered either phase-major over all row tiles ("data flow") or as independent (row tile,
// member) chains that a CTA interleaves ("chains"); either way, before a unit's inputs are loaded the
// producer acquires the arrival counters of the units that wrote them (sync[phase][row tile][member]),
// and every consumer warpgroup releases one arrival when its part of a unit is stored.  Every unit
// depends only on units earlier in some CTA's order, and all CTAs are resident, so the waits resolve;
// they are bounded nonetheless (ANI_STATUS_INTERNAL instead of a hung GPU).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"

namespace ani {
namespace tc {

constexpr int TM = ANI_TILE_ROWS;        // 128 rows per tile = two wgmma M = 64 slices
constexpr int TN_MAX = 256;              // columns of one accumulator
constexpr int TK = OPND_KB;              // 32 columns per K-block = one 64-byte swizzle row of 16-bit pieces
constexpr int ROW_BYTES = OPND_ROW_BYTES;        // 64
constexpr int GROUP_BYTES = 8 * ROW_BYTES;       // 8-row swizzle group = 512 B (descriptor stride byte offset)
constexpr int PARTS = OPND_PARTS;                // 2 (fp16) or 3 (bf16)
constexpr int A_PART_BYTES = OPND_PART_BYTES;    // 8 KB (one piece of one A K-block)
constexpr int A_BLOCK_BYTES = OPND_BLOCK_BYTES;  // 16 / 24 KB: [p1 | p2 (| p3)], contiguous in global memory
constexpr int STAGE_BYTES = A_BLOCK_BYTES + PARTS * TN_MAX * ROW_BYTES;  // 48 / 72 KB
constexpr int STAGES = ANI_OPND_FP16X2 ? 4 : 3;                         // 192 / 216 KB of the 227 KB
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;                 // + alignment of the ring
// warpgroup 0 is the producer (one issuing warp), warpgroups 1 and 2 the consumers.  The launch gives every thread 168
// registers; the producer warpgroup hands all but PROD_REGS back and the consumers take them (2 x 232 + 40 = 504 of the
// 512 per lane of a sub-partition): room for the 128-register accumulator and the epilogue's prefetched activations.
constexpr int NUM_CONSUMER_WARPS = 8, PROD_WARP = 0;
constexpr int THREADS = (NUM_CONSUMER_WARPS + 4) * 32;  // 384
constexpr int PROD_REGS = 40, CONS_REGS = 232;
constexpr int MAX_PHASES = 6;
constexpr int CHAIN_MAX_D = 8;
constexpr long long SPIN_LIMIT = 6000000000LL;  // ~3 s of clock64 ticks

enum { EPI_BIAS_CELU = 0, EPI_MUL_DCELU = 1, EPI_PLAIN = 2, EPI_HEAD = 3 };
// The hidden-layer activation (ani_mlp_model::activation), a compile-time parameter of the epilogues and kernels:
//   ACT_CELU  CELU(alpha) after bias: EPI_MUL_DCELU recovers CELU' from the stored activation itself.
//   ACT_GELU  exact-erf GELU, no biases.  GELU is not invertible, so the forward epilogues of layers 1 and 2 also store
//             d = GELU'(z) into the DERIVATIVE OPERAND, the same-shaped tiled operand directly behind C (d_offset),
//             and EPI_MUL_DCELU multiplies by that d.  |d| <= 1.13: stored at the value scale, no range check.
enum { ACT_CELU = ANI_ACT_CELU, ACT_GELU = ANI_ACT_GELU };

struct Species {
  const unsigned char* Bt;  // tiled B operand
  const float* bias;  // [N] (+ member * bias_mstride) or nullptr
  int K, N;
  int a_moff, c_moff, bias_mstride;  // per-member column offsets into A / C (multiples of 32)
  const float* w4;    // EPI_HEAD: final layer weights [M][N] and biases [M]
  const float* b4;
  // split-K over the members (layer-1 backward): all members share ONE B operand with b_kblocks
  // K-blocks, member m starts at K-block m * b_kb_moff.  0: one B operand per member.
  int b_kblocks, b_kb_moff;
  float acc_scale;  // 1 / (scale of A x scale of this B operand): multiplies the raw accumulator
};

struct Args {
  const unsigned char* A;       // tiled activation matrix [row tile][a_kblocks][p1 | p2 (| p3)]
  void* C;                      // tiled activation matrix (EPI_PLAIN: plain row-major float [rows][ldc])
  int a_kblocks, c_kblocks;     // 32-column blocks per row of A / C  (= leading dimension / 32)
  int ldc;                      // EPI_PLAIN only
  int members;                  // GEMMs per row tile
  const int32_t* layout_info;   // [4 + S + 1]: ..., first row tile of species s, total row tiles
  const int32_t* kblocks;       // optional list of live 32-wide K-blocks: [count, ids...]  (layer-1 forward)
  const int32_t* nblocks;       // optional list of live 32-wide column blocks of C          (layer-1 backward)
  int num_species;
  float alpha;
  // EPI_HEAD (layer 3 + final layer + gradient seed fused in the epilogue)
  float* e_member;              // [M][rows_cap]
  const int32_t* row_atom;      // [rows_cap], -1 for padding rows
  int rows_cap;
  int want_backward;
  int c_accumulate;             // EPI_PLAIN: C += tile (vector RED), C zeroed by the caller
  float out_scale;              // operand scale of a tiled C (OPND_SCALE_VALUE activations / OPND_SCALE_GRAD gradients)
  float y_inv_scale;            // EPI_MUL_DCELU: 1 / scale of the stored activation that C overwrites
  int32_t* status;              // ANI_STATUS_OPERAND_RANGE is raised here (may be NULL)
  int allow_narrow;             // short tile lists may split every accumulator into two column tiles (not EPI_HEAD)
  int win_idx, win_cnt;         // this launch covers window win_idx of win_cnt equal parts of every species' row tiles
  int b_compact;                // with `nblocks`: B holds ONLY the live column blocks, packed like a dense operand of
                                // nb_count * 32 rows (mlp.cu: k_zero_live_blocks builds it every step) -- one bulk copy
                                // per K-block instead of one 2 KB copy per live block and piece
  float member_scale[ANI_MAX_MEMBERS];
  Species sp[ANI_MAX_SPECIES];
};

// one launch: a single GEMM (n_phases = 1, sync = nullptr) or the phases of a whole MLP step
struct StepArgs {
  int n_phases;
  int epi[MAX_PHASES];    // epilogue of the phase (EPI_*)
  int chain;              // 0: phase-major list; 1: independent (row tile, member) chains
  int depth;              // chains: how many a CTA interleaves (0: all of its chains, in rounds of <= CHAIN_MAX_D)
  int32_t* sync;          // [MAX_PHASES][sync_stride][ANI_MAX_MEMBERS] arrivals, zeroed by the launcher
  int sync_stride;        // row tiles of the row capacity
  long long* trace;       // optional clock64 stamps [cta < 4][unit < 8][role 3][4] (ani_b200_debug_gemm_trace)
  Args ph[MAX_PHASES];
};

// ---- PTX wrappers -------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA bulk copy global -> shared, completion signalled on the mbarrier (complete_tx::bytes)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void red_add_v2(float* dst, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra.uni WAIT_DONE;\n\t"
      "bra.uni WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ int ld_acquire_gpu(const int32_t* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu(int32_t* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// generic-proxy writes of other CTAs (acquired through a counter) -> visible to this thread's bulk copies
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
// named barrier of one consumer warpgroup (ids 1, 2; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }
// per-thread register budget of the executing warpgroup (all four of its warps execute it)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// L2 prefetch of a contiguous global range (multiple of 16 bytes)
__device__ __forceinline__ void prefetch_l2(const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}

// bounded wait for `*counter >= need` (one thread); raises the status word instead of hanging
__device__ __forceinline__ void wait_counter(const int32_t* counter, int need, int32_t* status) {
  if (ld_acquire_gpu(counter) >= need) return;
  const long long t0 = clock64();
  while (ld_acquire_gpu(counter) < need) {
    if (clock64() - t0 > SPIN_LIMIT) {
      if (status) atomicOr(status, ANI_STATUS_INTERNAL);
      break;
    }
  }
}

// ---- wgmma -------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// shared-memory matrix descriptor: K-major, SWIZZLE_64B, 8-row groups 512 B apart
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);   // start address
  d |= (uint64_t)1 << 16;                        // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(GROUP_BYTES >> 4) << 32;       // stride byte offset between 8-row groups
  d |= (uint64_t)2 << 62;                        // SWIZZLE_64B
  return d;
}

#if ANI_OPND_FP16X2
#define ANI_WGMMA_AB "f16.f16"
#else
#define ANI_WGMMA_AB "bf16.bf16"
#endif
// D[64 x 64] += A[64 x 16] * B[64 x 16]^T (fp32 accumulate), both from shared memory
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." ANI_WGMMA_AB " "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db));
}
// CELU(x) = max(0,x) + min(0, alpha*(exp(x/alpha)-1)) with exp via ex2.approx (rel. error ~2^-22:
// the negative branch is bounded by alpha, so the absolute error is < 1e-8 for alpha = 0.1)
struct CeluConst {
  float alpha, inv_alpha, inv_alpha_log2e;
};
__device__ __forceinline__ float celu(float x, const CeluConst& c) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * c.inv_alpha_log2e));
  return x > 0.f ? x : fmaf(c.alpha, e, -c.alpha);
}
__device__ __forceinline__ float dcelu_from_out(float y, const CeluConst& c) {
  return y > 0.f ? 1.0f : fmaf(y, c.inv_alpha, 1.0f);
}
// GELU(x) = x Phi(x) (torch's approximate="none") and GELU'(x) = Phi(x) + x phi(x), from one erf and one exp.
// Phi = (1 + erf(x / sqrt 2)) / 2 cancels in the negative tail: its absolute error stays ~3e-8 there (2^-25 |x| in
// GELU), below what the 16-bit operand pieces keep of the values around it.
__device__ __forceinline__ void gelu_and_grad(float x, float& a, float& d) {
  const float cdf = fmaf(0.5f, erff(x * 0.70710678118654752f), 0.5f);
  float e;  // exp(-x^2 / 2) = 2^(-x^2 log2(e) / 2)
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * x * -0.72134752044448170f));
  a = x * cdf;
  d = fmaf(x * 0.39894228040143268f, e, cdf);
}
// byte offset of the derivative operand of a GELU model behind a tiled activation operand of c_kblocks 32-column
// blocks per row (include/ani_b200.h section 6)
__device__ __forceinline__ size_t d_offset(int rows_cap, int c_kblocks) {
  return (size_t)(rows_cap / TM) * c_kblocks * A_BLOCK_BYTES;
}
// running max of |v| in which a NaN sticks (fmaxf drops it): an inf/NaN operand piece turns the products into NaN,
// and that must raise ANI_STATUS_OPERAND_RANGE like any other value out of range
__device__ __forceinline__ float max_abs_nan(float m, float v) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(m), "f"(fabsf(v)));
  return r;
}

// ---- tile enumeration -----------------------------------------------------------------------
// Row tiles of one species are contiguous; tile t -> (species, row tile, member, n0, bn).
constexpr int MAX_BLOCKS = 64;         // ldx / 32 <= 64
struct TileMap {
  int first_rt[ANI_MAX_SPECIES + 1];   // first row tile of each species inside this launch's window
  int cnt_rt[ANI_MAX_SPECIES];         // row tiles of each species inside the window
  int ntn[ANI_MAX_SPECIES];            // N tiles per (row tile, member)
  int prefix[ANI_MAX_SPECIES + 1];     // exclusive prefix of tile counts
  int n_eff[ANI_MAX_SPECIES];          // columns actually computed (compacted when nblocks is given)
  int tn[ANI_MAX_SPECIES];             // columns per tile: TN_MAX, or half an accumulator for short lists
  int kb_count, nb_count;              // live K-blocks (-1: dense) / live column blocks (-1: dense)
  int kb[MAX_BLOCKS], nb[MAX_BLOCKS];
};

struct Tile {
  int s, rt, mem, n0, bn;
};

__device__ __forceinline__ void build_tile_map(const Args& a, TileMap& tm) {
  const int S = a.num_species;
  tm.kb_count = tm.nb_count = -1;
  if (a.kblocks) {
    tm.kb_count = min(a.kblocks[0], MAX_BLOCKS);
    for (int i = 0; i < tm.kb_count; ++i) tm.kb[i] = a.kblocks[1 + i];
  }
  if (a.nblocks) {
    tm.nb_count = min(a.nblocks[0], MAX_BLOCKS);
    for (int i = 0; i < tm.nb_count; ++i) tm.nb[i] = a.nblocks[1 + i];
  }
  const int wc = a.win_cnt > 1 ? a.win_cnt : 1, wi = a.win_cnt > 1 ? a.win_idx : 0;
  for (int s = 0; s < S; ++s) {
    const int f = a.layout_info[4 + s], nrt_all = a.layout_info[4 + s + 1] - f;
    const int lo = f + (int)((long long)nrt_all * wi / wc), hi = f + (int)((long long)nrt_all * (wi + 1) / wc);
    tm.first_rt[s] = lo;
    tm.cnt_rt[s] = hi - lo;
    tm.n_eff[s] = tm.nb_count >= 0 ? tm.nb_count * 32 : a.sp[s].N;
    tm.tn[s] = TN_MAX;
    tm.ntn[s] = (tm.n_eff[s] + TN_MAX - 1) / TN_MAX;
  }
  tm.first_rt[S] = a.layout_info[4 + S];
  auto count = [&]() {
    int run = 0;
    for (int s = 0; s < S; ++s) {
      tm.prefix[s] = run;
      run += tm.cnt_rt[s] * a.members * tm.ntn[s];
    }
    tm.prefix[S] = run;
    return run;
  };
  const int wide = count();
  // Short lists (less than half a wave of 256-column tiles: 1 k-atom systems, multi-GPU shards): split every
  // accumulator into two column tiles -- twice the CTAs at work, each with half the main loop and half the epilogue,
  // which is what the latency of the layer chain is made of.  (Tiles never straddle a packed 256-row B tile.)
  // tests/test_gpu_mlp.py restates this rule (layer1_forward_tiles) to assert which side its cases run: change both.
  if (a.allow_narrow && wide > 0 && 2 * wide <= (int)gridDim.x) {
    for (int s = 0; s < S; ++s) {
      tm.tn[s] = tm.n_eff[s] > TN_MAX ? TN_MAX / 2 : max(32, ((tm.n_eff[s] / 32 + 1) / 2) * 32);
      tm.ntn[s] = (tm.n_eff[s] + tm.tn[s] - 1) / tm.tn[s];
    }
    count();
  }
}

__device__ __forceinline__ Tile make_tile(const TileMap& tm, int s, int rt, int mem, int nt) {
  Tile x;
  x.s = s;
  x.rt = rt;
  x.mem = mem;
  x.n0 = nt * tm.tn[s];
  x.bn = min(tm.tn[s], tm.n_eff[s] - x.n0);
  return x;
}

__device__ __forceinline__ Tile decode_tile(const Args& a, const TileMap& tm, int t) {
  int s = 0;
  while (t >= tm.prefix[s + 1]) ++s;
  const int local = t - tm.prefix[s];
  const int ntn = tm.ntn[s];
  const int rm = local / ntn;
  return make_tile(tm, s, tm.first_rt[s] + rm / a.members, rm % a.members, local % ntn);
}

// ---- split of two adjacent (already scaled) fp32 values into PARTS packed 16-bit pairs (low half = a)
__device__ __forceinline__ void split_pair(float a, float b, uint32_t (&w)[PARTS]) {
#if ANI_OPND_FP16X2
  __half2 h = __floats2half2_rn(a, b);
  w[0] = *reinterpret_cast<uint32_t*>(&h);
  const float2 f = __half22float2(h);
  h = __floats2half2_rn(a - f.x, b - f.y);
  w[1] = *reinterpret_cast<uint32_t*>(&h);
#else
#pragma unroll
  for (int p = 0; p < PARTS; ++p) {
    __nv_bfloat162 q = __floats2bfloat162_rn(a, b);
    w[p] = *reinterpret_cast<uint32_t*>(&q);
    a -= __uint_as_float(w[p] << 16);
    b -= __uint_as_float(w[p] & 0xffff0000u);
  }
#endif
}
// sum of the pieces of one packed pair (smallest piece first) -> 2 floats (still times the operand scale)
__device__ __forceinline__ float2 join_pair(const uint32_t (&w)[PARTS]) {
  float lo = 0.f, hi = 0.f;
#pragma unroll
  for (int p = PARTS - 1; p >= 0; --p) {
#if ANI_OPND_FP16X2
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[p]));
    lo += f.x;
    hi += f.y;
#else
    lo += __uint_as_float(w[p] << 16);
    hi += __uint_as_float(w[p] & 0xffff0000u);
#endif
  }
  return make_float2(lo, hi);
}

// Transpose of 4 x 4 words inside a quad of lanes: on entry lane q holds x[j] = word q of 16-byte chunk j; on exit
// it holds x[t] = word t of chunk q.  (The wgmma accumulator gives a thread two adjacent columns of every 8-column
// chunk; the tiled layout wants whole 16-byte chunks per row.)
__device__ __forceinline__ void quad_transpose(uint32_t (&x)[4], int lane) {
  const int q = lane & 3;
  uint32_t out[4] = {x[0], x[0], x[0], x[0]};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int want = (q + k) & 3;  // the receiver (q + k) & 3 ... gets it from the sender (q - k) & 3
    const uint32_t send = want == 0 ? x[0] : want == 1 ? x[1] : want == 2 ? x[2] : x[3];
    const int src = (q - k) & 3;
    const uint32_t got = __shfl_sync(ANI_FULL_MASK, send, (lane & ~3) | src);
#pragma unroll
    for (int t = 0; t < 4; ++t) out[t] = t == src ? got : out[t];
  }
#pragma unroll
  for (int t = 0; t < 4; ++t) x[t] = out[t];
}

// ---- work lists ----------------------------------------------------------------------------
struct Unit {
  int p;
  Tile tl;
};

// The n-th unit of a CTA.  Phase-major: unit c, c + G, ... of the concatenated phase lists.  Chains: chain
// (row tile, member) ids c, c + G, ... in rounds of D chains; inside a round phase-major, chain-minor.
struct Walk {
  const StepArgs* F;
  const TileMap* tms;
  int G, c;
  // phase-major
  int u, total;
  // chains
  int D, M, num_chains, round, p, j, nt;
  __device__ __forceinline__ void init(const StepArgs& F_, const TileMap* tms_, int G_, int c_) {
    F = &F_;
    tms = tms_;
    G = G_;
    c = c_;
    u = c_ - G_;
    total = 0;
    for (int q = 0; q < F_.n_phases; ++q) total += tms_[q].prefix[F_.ph[q].num_species];
    const TileMap& t0 = tms_[0];
    const int S = F_.ph[0].num_species;
    int rts = 0;
    for (int s = 0; s < S; ++s) rts += t0.cnt_rt[s];
    M = F_.ph[0].members;
    num_chains = rts * M;
    const int per_cta = (num_chains - c_ + G_ - 1) / G_;
    D = F_.depth > 0 ? min(F_.depth, CHAIN_MAX_D) : max(1, min(CHAIN_MAX_D, per_cta));
    round = 0;
    p = 0;
    j = 0;
    nt = -1;
  }
  // CHAIN: F->chain, known at compile time (the producer warp: no registers for the state of the other order)
  __device__ __forceinline__ bool next(Unit& x) { return F->chain ? next<true>(x) : next<false>(x); }
  template <bool CHAIN>
  __device__ __forceinline__ bool next(Unit& x) {
    if (!CHAIN) {
      u += G;
      if (u >= total) return false;
      int t = u, q = 0;
      while (t >= tms[q].prefix[F->ph[q].num_species]) t -= tms[q].prefix[F->ph[q].num_species], ++q;
      x.p = q;
      x.tl = decode_tile(F->ph[q], tms[q], t);
      return true;
    }
    while (true) {
      const int ch = c + (round * D + j) * G;
      if (round * D * G + c >= num_chains) return false;
      if (ch < num_chains) {
        // chain -> (species, row tile, member)
        const TileMap& t0 = tms[0];
        int r = ch / M, s = 0;
        while (r >= t0.cnt_rt[s]) r -= t0.cnt_rt[s], ++s;
        const int ntn = tms[p].ntn[s];
        if (++nt < ntn) {
          x.p = p;
          x.tl = make_tile(tms[p], s, tms[p].first_rt[s] + r, ch % M, nt);
          return true;
        }
      }
      nt = -1;
      if (++j == D) {
        j = 0;
        if (++p == F->n_phases) {
          p = 0;
          ++round;
        }
      }
    }
  }
};

// arrival counter of (phase, row tile, member)
__device__ __forceinline__ int32_t* counter(const StepArgs& F, int p, int rt, int m) {
  return F.sync + ((size_t)p * F.sync_stride + rt) * ANI_MAX_MEMBERS + m;
}
// the inputs of unit (p, tile) were written by phase p - 1 of the same row tile: the members whose columns it reads
// (a member group in a grouped layer-1 backward); each of their units owes one arrival per consumer warpgroup
__device__ __forceinline__ void wait_inputs(const StepArgs& F, const TileMap* tms, int p, const Tile& tl) {
  if (!F.sync || p == 0) return;
  const int G = F.ph[0].members / F.ph[p].members;
  const int need = 2 * tms[p - 1].ntn[tl.s];
  for (int m = tl.mem * G; m < (tl.mem + 1) * G; ++m) wait_counter(counter(F, p - 1, tl.rt, m), need, F.ph[p].status);
}

// ---- epilogue of one consumer warpgroup: 64 rows x bn columns straight from the accumulator registers ----
// Register i of 64-column slice c holds row 16 * warp + lane / 4 + 8 * ((i >> 1) & 1), column
// 64 c + 8 (i >> 2) + 2 (lane & 3) + (i & 1).
template <int EPI, int ACT>
__device__ __forceinline__ void tile_epilogue(const Args& args, const TileMap& tm, const Tile& tl, float (&acc)[4][32],
                                              int wg, int lane, int warp_in_wg, float& omax) {
  const Species& sp = args.sp[tl.s];
  const CeluConst cc{args.alpha, 1.0f / args.alpha, 1.4426950408889634f / args.alpha};
  const int q = lane & 3;
  const int r0 = 64 * wg + 16 * warp_in_wg + (lane >> 2);  // rows r0 and r0 + 8 of the tile
  const float acc_scale = sp.acc_scale;
  constexpr bool GELU = ACT == ACT_GELU;
  const bool tiled_out = EPI != EPI_PLAIN && (EPI != EPI_HEAD || args.want_backward);
  unsigned char* ct = reinterpret_cast<unsigned char*>(args.C) +
                      ((size_t)tl.rt * args.c_kblocks + (size_t)(tl.mem * sp.c_moff + tl.n0) / TK) * A_BLOCK_BYTES;
  // GELU: where d = GELU'(z) of these columns is stored (EPI_BIAS_CELU, only for a backward) and read (EPI_MUL_DCELU)
  unsigned char* dt = GELU ? ct + d_offset(args.rows_cap, args.c_kblocks) : nullptr;
  const bool store_d = GELU && EPI == EPI_BIAS_CELU && args.want_backward;
  const float* bias = !GELU && (EPI == EPI_BIAS_CELU || EPI == EPI_HEAD) ? sp.bias + (size_t)tl.mem * sp.bias_mstride + tl.n0
                                                                         : nullptr;
  const float* w4 = EPI == EPI_HEAD ? sp.w4 + (size_t)tl.mem * sp.N : nullptr;
  float e_acc[2] = {0.f, 0.f}, seed[2] = {0.f, 0.f};
  bool row_valid[2] = {false, false};
  if (EPI == EPI_HEAD) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      row_valid[h] = args.row_atom[tl.rt * TM + r0 + 8 * h] >= 0;
      seed[h] = row_valid[h] ? args.member_scale[tl.mem] : 0.f;
    }
  }
  const int ngroups = tl.bn / 32;
  // EPI_MUL_DCELU: the stored activation (GELU: the stored derivative) of the next (32-column group, row half) is loaded
  // before the current one is computed and stored in its place.  (Loads may not pass stores into the same buffer, so
  // without this every step would wait for a full global round trip.)  [step parity][piece]: chunk q of every piece
  // of the row
  uint4 ybuf[2][PARTS];
  auto load_y = [&](int g, int h, uint4 (&dst)[PARTS]) {
    const unsigned char* blk = (GELU ? dt : ct) + (size_t)g * A_BLOCK_BYTES + swz_off(r0 + 8 * h, q);
#pragma unroll
    for (int p = 0; p < PARTS; ++p) dst[p] = *reinterpret_cast<const uint4*>(blk + p * A_PART_BYTES);
  };
  if (EPI == EPI_MUL_DCELU) load_y(0, 0, ybuf[0]);
#pragma unroll
  for (int g = 0; g < TN_MAX / 32; ++g) {
    if (g >= ngroups) break;
    const int c = g >> 1, ib = (g & 1) * 16;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + 8 * h;
      if (EPI == EPI_MUL_DCELU) {
        if (h == 0)
          load_y(g, 1, ybuf[1]);
        else if (g + 1 < ngroups)
          load_y(g + 1, 0, ybuf[0]);
      }
      // stored activation of this row's 32 columns (EPI_MUL_DCELU), transposed to pairs
      uint32_t yw[PARTS][4];
      if (EPI == EPI_MUL_DCELU) {
#pragma unroll
        for (int p = 0; p < PARTS; ++p) {
          const uint4 v = ybuf[h][p];
          yw[p][0] = v.x, yw[p][1] = v.y, yw[p][2] = v.z, yw[p][3] = v.w;
          quad_transpose(yw[p], lane);
        }
      }
      uint32_t w[PARTS][4], dw[PARTS][4];
      float o[4][2], od[2];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = 32 * g + 8 * j + 2 * q;  // column inside the tile
        float2 b2 = make_float2(0.f, 0.f), w2 = make_float2(0.f, 0.f), y2 = make_float2(0.f, 0.f);
        if (!GELU && (EPI == EPI_BIAS_CELU || EPI == EPI_HEAD)) b2 = __ldg(reinterpret_cast<const float2*>(bias + col));
        if (EPI == EPI_HEAD) w2 = __ldg(reinterpret_cast<const float2*>(w4 + col));
        if (EPI == EPI_MUL_DCELU) {
          uint32_t pw[PARTS];
#pragma unroll
          for (int p = 0; p < PARTS; ++p) pw[p] = yw[p][j];
          y2 = join_pair(pw);
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float v = acc[c][ib + 4 * j + 2 * h + e] * acc_scale;
          const float bb = e ? b2.y : b2.x, ww = e ? w2.y : w2.x, yy = e ? y2.y : y2.x;
          if (GELU && EPI == EPI_BIAS_CELU) {
            float d;
            gelu_and_grad(v, v, d);
            od[e] = d * args.out_scale;
          } else if (GELU && EPI == EPI_MUL_DCELU) {
            v *= yy * args.y_inv_scale;
          } else if (GELU && EPI == EPI_HEAD) {
            float a, d;
            gelu_and_grad(v, a, d);
            e_acc[h] = fmaf(a, ww, e_acc[h]);
            v = seed[h] * ww * d;
          } else if (EPI == EPI_BIAS_CELU) {
            v = celu(v + bb, cc);
          } else if (EPI == EPI_MUL_DCELU) {
            v *= dcelu_from_out(yy * args.y_inv_scale, cc);
          } else if (EPI == EPI_HEAD) {
            const float a = celu(v + bb, cc);
            e_acc[h] = fmaf(a, ww, e_acc[h]);
            v = seed[h] * ww * dcelu_from_out(a, cc);
          }
          if (EPI != EPI_PLAIN) {
            v *= args.out_scale;
            omax = max_abs_nan(omax, v);
          }
          o[j][e] = v;
        }
        if (tiled_out) {
          uint32_t pw[PARTS];
          split_pair(o[j][0], o[j][1], pw);
#pragma unroll
          for (int p = 0; p < PARTS; ++p) w[p][j] = pw[p];
        }
        if (store_d) {
          uint32_t pw[PARTS];
          split_pair(od[0], od[1], pw);
#pragma unroll
          for (int p = 0; p < PARTS; ++p) dw[p][j] = pw[p];
        }
      }
      if (EPI == EPI_PLAIN) {
        float* cplain = reinterpret_cast<float*>(args.C) + (size_t)(tl.rt * TM + row) * args.ldc + (size_t)tl.mem * sp.c_moff;
        // compacted column blocks map back to their place: group g is live block n0/32 + g
        const int col0 = tm.nb_count >= 0 ? tm.nb[tl.n0 / 32 + g] * 32 : tl.n0 + g * 32;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float* dst = cplain + col0 + 8 * j + 2 * q;
          if (args.c_accumulate)
            red_add_v2(dst, o[j][0], o[j][1]);
          else
            *reinterpret_cast<float2*>(dst) = make_float2(o[j][0], o[j][1]);
        }
      } else if (tiled_out) {
        unsigned char* blk = ct + (size_t)g * A_BLOCK_BYTES + swz_off(row, q);
#pragma unroll
        for (int p = 0; p < PARTS; ++p) {
          quad_transpose(w[p], lane);
          *reinterpret_cast<uint4*>(blk + p * A_PART_BYTES) = make_uint4(w[p][0], w[p][1], w[p][2], w[p][3]);
        }
        if (store_d) {
          unsigned char* dblk = dt + (size_t)g * A_BLOCK_BYTES + swz_off(row, q);
#pragma unroll
          for (int p = 0; p < PARTS; ++p) {
            quad_transpose(dw[p], lane);
            *reinterpret_cast<uint4*>(dblk + p * A_PART_BYTES) = make_uint4(dw[p][0], dw[p][1], dw[p][2], dw[p][3]);
          }
        }
      }
    }
  }
  if (EPI == EPI_HEAD) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float e = e_acc[h];
      e += __shfl_xor_sync(ANI_FULL_MASK, e, 1);
      e += __shfl_xor_sync(ANI_FULL_MASK, e, 2);
      if (q == 0)
        args.e_member[(size_t)tl.mem * args.rows_cap + tl.rt * TM + r0 + 8 * h] = row_valid[h] ? e + sp.b4[tl.mem] : 0.f;
    }
  }
}

// ---- the kernel -----------------------------------------------------------------------------
// ACT: the activation of the model (ACT_CELU / ACT_GELU), one instance each
template <int ACT>
__global__ void __launch_bounds__(THREADS, 1) k_gemm_wg(const __grid_constant__ StepArgs F) {
  extern __shared__ unsigned char smem_raw[];
  // 1024-byte aligned ring (swizzle groups are 8 rows x 64 B)
  unsigned char* smem = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  __shared__ TileMap tms[MAX_PHASES];
  __shared__ __align__(8) uint64_t full[STAGES], empty[STAGES];
  // role and loop bounds broadcast from lane 0: provably warp-uniform, so ptxas keeps the wgmma issue asynchronous
  const int warp = __shfl_sync(ANI_FULL_MASK, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  auto stamp = [&](int tile_local, int role, int slot) {
    if (F.trace && blockIdx.x < 4 && tile_local < 8)
      F.trace[(((size_t)blockIdx.x * 8 + tile_local) * 3 + role) * 4 + slot] = clock64();
  };
  if (threadIdx.x < F.n_phases) build_tile_map(F.ph[threadIdx.x], tms[threadIdx.x]);
  if (threadIdx.x == 32) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);                     // the expect_tx arrival of the producer lane (+ the bytes)
      mbar_init(&empty[i], NUM_CONSUMER_WARPS);   // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  // programmatic dependent launch: the next kernel of the stream may start scheduling its CTAs from here on;
  // everything above did not touch data the previous kernel writes (layout_info / block lists are older),
  // everything below may: wait for the previous grid to complete and flush.  No-ops in a plain launch.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (warp < 4) {
    setmaxnreg_dec<PROD_REGS>();
    if (warp != PROD_WARP) return;
    // ================================ producer (TMA) ================================
    // one loop per list order: the walk state of the other order would not fit the producer's registers
    auto produce = [&](auto chain) {
      Walk walk;
      walk.init(F, tms, (int)gridDim.x, (int)blockIdx.x);
      uint32_t stage = 0, phase = 0;
      int tloc = 0;
      Unit un;
      while (walk.template next<decltype(chain)::value>(un)) {
        const Args& args = F.ph[un.p];
        const TileMap& tm = tms[un.p];
        const Tile& tl = un.tl;
        const Species& sp = args.sp[tl.s];
        const int nkb = tm.kb_count >= 0 ? tm.kb_count : (sp.K + TK - 1) / TK;
        if (lane == 0) {
          stamp(tloc, 0, 0);
          wait_inputs(F, tms, un.p, tl);
          if (F.sync) fence_proxy_async_all();
          // the stored activation (GELU: derivative) the dCELU epilogue reads: contiguous 32-column blocks of this tile,
          // on their way to L2 while the main loop runs
          if (F.epi[un.p] == EPI_MUL_DCELU)
            prefetch_l2(static_cast<const unsigned char*>(args.C) +
                            (ACT == ACT_GELU ? d_offset(args.rows_cap, args.c_kblocks) : (size_t)0) +
                            ((size_t)tl.rt * args.c_kblocks + (size_t)(tl.mem * sp.c_moff + tl.n0) / TK) * A_BLOCK_BYTES,
                        (uint32_t)(tl.bn / TK) * A_BLOCK_BYTES);
        }
        __syncwarp();
        const int nkb_all = sp.b_kb_moff ? sp.b_kblocks : (sp.K + TK - 1) / TK;  // K-blocks of the stored B operand
        const int kb_boff = tl.mem * sp.b_kb_moff;                               // split-K: this member's first K-block
        // A: [row tile][32-column block][p1 | p2 | p3]; this GEMM starts at column member * a_moff
        const unsigned char* At =
            args.A + ((size_t)tl.rt * args.a_kblocks + (size_t)(tl.mem * sp.a_moff) / TK) * A_BLOCK_BYTES;
        // B: [member][n tile][k block][p1 bn x 64 B | p2 | p3]
        const unsigned char* Bm = sp.Bt + (sp.b_kb_moff ? (size_t)0 : (size_t)tl.mem * sp.N * nkb_all * (PARTS * ROW_BYTES));
        const uint32_t b_bytes = (uint32_t)tl.bn * ROW_BYTES;  // one piece of the tile's B rows
        const bool dense = tm.nb_count < 0 || args.b_compact;
        // the packed B tile this one lies in
        const int n0p = tl.n0 / TN_MAX * TN_MAX, bnp = min(TN_MAX, (args.b_compact ? tm.n_eff[tl.s] : sp.N) - n0p);
        // gathered column blocks (layer-1 backward): lane -> (live block q, piece)
        const int gq = lane / PARTS, gpart = lane % PARTS;
        size_t g_src = 0;
        int g_bns = 0;
        const bool g_active = !dense && lane < PARTS * (tl.bn / 32);
        if (g_active) {
          const int row0 = tm.nb[tl.n0 / 32 + gq] * 32;
          const int n0s = row0 / TN_MAX * TN_MAX;
          g_bns = min(TN_MAX, sp.N - n0s);
          g_src = (size_t)n0s * nkb_all * (PARTS * ROW_BYTES) + (size_t)(row0 - n0s) * ROW_BYTES +
                  (size_t)gpart * g_bns * ROW_BYTES;
        }
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          unsigned char* st = smem + stage * STAGE_BYTES;
          const int kbi = tm.kb_count >= 0 ? tm.kb[kb] : kb;
          const int kbb = kbi + kb_boff;
          if (lane == 0) {
            mbar_arrive_expect_tx(&full[stage], A_BLOCK_BYTES + PARTS * b_bytes);
            bulk_g2s(st, At + (size_t)kbi * A_BLOCK_BYTES, A_BLOCK_BYTES, &full[stage]);
            if (dense) {
              if (tl.bn == bnp) {  // the pieces are adjacent in global memory and in shared memory: one copy
                bulk_g2s(st + A_BLOCK_BYTES, Bm + ((size_t)tl.n0 * nkb_all + (size_t)kbb * tl.bn) * (PARTS * ROW_BYTES),
                         PARTS * b_bytes, &full[stage]);
              } else {             // a column tile inside a packed 256-row B tile: one copy per piece
#pragma unroll
                for (int p = 0; p < PARTS; ++p)
                  bulk_g2s(st + A_BLOCK_BYTES + p * b_bytes,
                           Bm + ((size_t)n0p * nkb_all + (size_t)kbb * bnp) * (PARTS * ROW_BYTES) +
                               (size_t)p * bnp * ROW_BYTES + (size_t)(tl.n0 - n0p) * ROW_BYTES,
                           b_bytes, &full[stage]);
              }
            }
          }
          __syncwarp();
          if (g_active)
            bulk_g2s(st + A_BLOCK_BYTES + gpart * b_bytes + gq * 32 * ROW_BYTES,
                     Bm + g_src + (size_t)kbb * g_bns * (PARTS * ROW_BYTES), 32 * ROW_BYTES, &full[stage]);
          __syncwarp();
          if (lane == 0 && kb == 0) stamp(tloc, 0, 1);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
        if (lane == 0) stamp(tloc, 0, 2);
        ++tloc;
      }
    };
    if (F.chain)
      produce(std::true_type{});
    else
      produce(std::false_type{});
    return;
  }

  // ================================ consumers ================================
  setmaxnreg_inc<CONS_REGS>();
  Walk walk;
  walk.init(F, tms, (int)gridDim.x, (int)blockIdx.x);
  const int wg = (warp >> 2) - 1, warp_in_wg = warp & 3;
  const bool leader = (threadIdx.x & 127) == 0;
  uint32_t stage = 0, phase = 0;
  float omax = 0.f;  // largest |scaled value| this thread handed to the half-precision split
  int tloc = 0;
  Unit un;
  while (__shfl_sync(ANI_FULL_MASK, (int)walk.next(un), 0)) {
    const Args& args = F.ph[un.p];
    const TileMap& tm = tms[un.p];
    const Tile& tl = un.tl;
    const Species& sp = args.sp[tl.s];
    const int nkb = __shfl_sync(ANI_FULL_MASK, tm.kb_count >= 0 ? tm.kb_count : (sp.K + TK - 1) / TK, 0);
    const int bn = tl.bn;
    const uint32_t b_bytes = (uint32_t)bn * ROW_BYTES;
    // 64-column slices of the accumulator.  A 32-column remainder is computed as a whole slice: its upper half reads
    // the rows that follow in the stage (never past it, bn <= 224 then) into accumulator columns nobody reads.
    const int nsl = __shfl_sync(ANI_FULL_MASK, (bn + 63) / 64, 0);
    if (wg == 0 && leader) stamp(tloc, 1, 0);
    float acc[4][32];
    // NSL = nsl at compile time: a K-block's products are then one branch-free commit group (a run-time slice count
    // inside the group split it into one wgmma group per branch, so wgmma.wait_group 1 waited for all of them).  Only
    // the NSL slices the epilogue reads are zeroed: zeros in the others would be copied into them at every exit.
    auto main_loop = [&](auto nsl_) {
      constexpr int NSL = decltype(nsl_)::value;
#pragma unroll
      for (int c = 0; c < NSL; ++c)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
      uint32_t prev = 0;
#pragma unroll 1
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full[stage], phase);
        if (wg == 0 && leader && kb == 0) stamp(tloc, 1, 1);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + wg * (64 / 8) * GROUP_BYTES;  // this warpgroup's rows
        const uint32_t sb = smem_u32(smem + stage * STAGE_BYTES) + A_BLOCK_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TK / 16; ++k) {
          const uint32_t adv = 32u * k;  // 16 pieces = 32 B along the swizzle row
          uint64_t da[PARTS];
#pragma unroll
          for (int p = 0; p < PARTS; ++p) da[p] = make_desc(sa + p * A_PART_BYTES + adv);
#pragma unroll
          for (int c = 0; c < NSL; ++c) {
            uint64_t db[PARTS];
#pragma unroll
            for (int p = 0; p < PARTS; ++p) db[p] = make_desc(sb + p * b_bytes + c * (64 / 8) * GROUP_BYTES + adv);
            auto mma = [&](int pa, int pb) { wgmma_n64(acc[c], da[pa], db[pb]); };
            // smallest terms first
#if ANI_OPND_FP16X2
            mma(1, 0);
            mma(0, 1);
            mma(0, 0);
#else
            mma(2, 0);
            mma(0, 2);
            mma(1, 1);
            mma(1, 0);
            mma(0, 1);
            mma(0, 0);
#endif
          }
        }
        wgmma_commit();
        // the previous K-block's products have retired: its slot goes back to the producer
        wgmma_wait<1>();
        if (kb > 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      if (nkb > 0 && lane == 0) mbar_arrive(&empty[prev]);
    };
    switch (nsl) {
      case 1: main_loop(std::integral_constant<int, 1>{}); break;
      case 2: main_loop(std::integral_constant<int, 2>{}); break;
      case 3: main_loop(std::integral_constant<int, 3>{}); break;
      default: main_loop(std::integral_constant<int, 4>{}); break;
    }
    if (wg == 0 && leader) stamp(tloc, 1, 2);
    // the stored activation of EPI_MUL_DCELU was written by other CTAs: acquire its counters in this warpgroup too
    if (F.sync && F.epi[un.p] == EPI_MUL_DCELU) {
      if (leader) wait_inputs(F, tms, un.p, tl);
      wg_bar(wg);
    }
    switch (F.epi[un.p]) {
      case EPI_BIAS_CELU: tile_epilogue<EPI_BIAS_CELU, ACT>(args, tm, tl, acc, wg, lane, warp_in_wg, omax); break;
      case EPI_MUL_DCELU: tile_epilogue<EPI_MUL_DCELU, ACT>(args, tm, tl, acc, wg, lane, warp_in_wg, omax); break;
      case EPI_HEAD: tile_epilogue<EPI_HEAD, ACT>(args, tm, tl, acc, wg, lane, warp_in_wg, omax); break;
      default: tile_epilogue<EPI_PLAIN, ACT>(args, tm, tl, acc, wg, lane, warp_in_wg, omax); break;
    }
    // one release per warpgroup and unit: its 64 rows of the tile are stored
    if (F.sync && un.p + 1 < F.n_phases) {
      wg_bar(wg);
      if (leader) {
        __threadfence();
        red_release_gpu(counter(F, un.p, tl.rt, tl.mem), 1);
      }
    }
    if (wg == 0 && leader) stamp(tloc, 2, 0);
    ++tloc;
  }
  const Args& a0 = F.ph[0];
  if (ANI_OPND_FP16X2 && a0.status && !(omax <= OPND_HALF_MAX)) atomicOr(a0.status, ANI_STATUS_OPERAND_RANGE);
}

}  // namespace tc
}  // namespace ani
