// The whole ensemble MLP of a step with every intermediate resident in shared memory (sm_90a, 2 x fp16 build).
//
// A chain is one (128-row tile, member) pair.  One persistent CTA per SM runs whole chains, each as six phases back to
// back, and hands every layer's output to the next layer through a resident region R of shared memory instead of
// global memory:
//
//   phase  A operand                B operand (ring)               epilogue
//   0      x live K-blocks (ring)   W1_m                           a1 = CELU(.)  -> R and act1 (for phase 4)
//   1      R                        W2_m                           a2 = CELU(.)  -> R and act2 (for phase 3)
//   2      R                        W3_m                           head: e_member; G3 -> R
//   3      R                        W3_m^T                         G2 = (.) * CELU'(act2) -> R
//   4      R                        W2_m^T                         G1 = (.) * CELU'(act1) -> R
//   5      R                        W1^T (member m's K-blocks),    dE/dAEV: vector REDs into dx (M > 1) or stores
//                                   <= 256 live columns per tile
//
// R is 8 K-blocks (256 columns) in the tiled-operand layout of common.cuh, so the wgmma descriptors of gemm_tc.cuh read
// it unchanged.  Consumer warpgroup w reads and writes only rows 64w .. 64w+63 of R: a phase's output goes into R after
// the warpgroup's last wgmma of that phase has retired, and a warpgroup barrier after fence.proxy.async makes it
// visible to the next phase's wgmma.  The only inputs are x (an earlier launch) and the weights, so nothing waits on
// another CTA: the producer streams B (and x in phase 0) ahead across phase and chain boundaries, limited only by the
// free ring slots.
//
// Main loop: one wgmma per K-step, product and B slot, as wide as the slot's rows (m64n128k16, or n32 / n64 / n96 for
// the remainder of the phase's columns), so A is read from shared memory once per 128 columns and no MMA runs on
// padding.  The products keep the order a2b1, a1b2, a1b1, so every output element sees the same sums as with 64-column
// slices.  Epilogue stores into R: stmatrix.x4 per (32-column group, row half, piece), matrix j = chunk j of the
// group, each lane addressing one swizzled 16-byte row.
//
// act1 / act2 (read back for CELU' by phases 4 / 3) leave R by bulk copy.  Once the threads of a warpgroup have stored
// their rows of phase 0 / 1, run fence.proxy.async.shared::cta and met at the warpgroup barrier, one of them (the
// copier) issues cp.async.bulk.global.shared::cta for the warpgroup's 4 KB of every K-block and piece.  The fence
// and the barrier order every thread's generic stores into R before the copier's async-proxy reads of R, as for wgmma.
// The copier waits with cp.async.bulk.wait_group.read 0 before the barrier in front of the next epilogue (phases 1, 2),
// so R is not overwritten while a copy still reads it.  Before the barrier in front of phase 3's epilogue it waits with
// cp.async.bulk.wait_group 0: the copies of a1 and a2 are complete, and completion makes their writes visible to the
// copier.  bar.sync then orders them before every later memory access of the warpgroup's other threads (the barrier
// is a CTA-scope synchronisation in the PTX memory model, and causality order is transitive), so phases 3 and 4 read
// the finished values.  They load with ld.global.cg: nothing of these lines was cached in this SM's L1 earlier in the
// launch, and .cg leaves no room for a stale line either way.  Every copy of a chain is complete by its phase 3, so
// none is in flight when the next chain's phase 0 overwrites R or when the CTA exits.
//
// GELU models (ACT_GELU): phases 0 / 1 store a = GELU(z) into R and d = GELU'(z) into act1 / act2, each thread the
// words it computed with plain stores (exactly the words its load_y reads back in phases 4 / 3, so program order alone
// makes them visible); nothing reads a1 / a2 after the forward phases, and there are no bulk copies.  Phases 3 / 4
// multiply by d, the head computes GELU and GELU' from registers, and no bias is loaded.
//
// Shared memory: R 128 KB + a ring of six 16 KB slots + 1 KB alignment = 230,400 B.  A K-block takes one slot for
// the x block of phase 0 and one per 128 rows of B.
// The 3 x bf16 build would need 192 KB for R and does not compile this kernel.
#pragma once
#include "gemm_tc.cuh"

namespace ani {
namespace tc {

constexpr int RES_KBLOCKS = 8;   // widest layer of an eligible model: 256 columns
constexpr int RES_PHASES = 6;
#if ANI_OPND_FP16X2
constexpr int RES_BYTES = RES_KBLOCKS * A_BLOCK_BYTES;                  // 128 KB
// Ring of 16 KB slots: one x K-block, or 128 rows of a B K-block ([p1 128 x 64 B | p2 128 x 64 B]).  A K-block takes
// 1-3 slots, so phases 1-5 keep two K-blocks of B in flight where 48 KB stages would keep one.
constexpr int RES_SLOT_BYTES = A_BLOCK_BYTES;
constexpr int RES_SLOTS = 6;
constexpr int RES_HALF = TN_MAX / 2;                                    // B rows per slot
constexpr int RES_SMEM_BYTES = RES_BYTES + RES_SLOTS * RES_SLOT_BYTES + 1024;
static_assert(RES_SMEM_BYTES <= 232448 - 1024, "resident MLP: shared memory over the per-block limit");
static_assert(PARTS * RES_HALF * ROW_BYTES == RES_SLOT_BYTES, "a slot holds 128 B rows of every piece");
#endif

struct ResSpecies {
  const unsigned char* B[RES_PHASES];  // tiled B operands of the phases: W1, W2, W3, W3^T, W2^T per member; W1^T shared
  const float* bias[3];                // [M][h] per layer
  const float* w4;                     // [M][h3]
  const float* b4;                     // [M]
  int h1, h2, h3;
  float acc_scale[RES_PHASES];         // 1 / (scale of A x scale of B) of every phase
};

struct ResArgs {
  const unsigned char* x;              // tiled AEV operand, kbx K-blocks per row tile
  unsigned char* act1;                 // tiled a1 [row tile][kb1], member m at column m * h1
  unsigned char* act2;                 // tiled a2 [row tile][kb2]
  float* dx;                           // plain [rows_cap][ldx]
  float* e_member;                     // [M][rows_cap]
  const int32_t* layout_info;          // [4 + S + 1]: ..., first row tile of species s, total row tiles
  const int32_t* row_atom;             // [rows_cap], -1 for padding rows
  const int32_t* blocks;               // live 32-column AEV blocks [count, ids...] or nullptr (all live)
  int kbx, kb1, kb2, ldx, rows_cap, members, num_species;
  int b_compact;                       // with `blocks`: B[5] holds only the live column blocks (mlp.cu b1_compact)
  float alpha;
  int32_t* status;
  int order[ANI_MAX_SPECIES];          // species by decreasing chain length: the longest chains start first
  float member_scale[ANI_MAX_MEMBERS];
  ResSpecies sp[ANI_MAX_SPECIES];
  // per-member slabs (k_mlp_resident<true>): the chains of a row tile are those of the n_chain_members members
  // member_of[0..), and phase 5 stores member m's dE/dAEV into dx + m * slab_stride instead of reducing into dx
  long long slab_stride;
  int n_chain_members;
  int member_of[ANI_MAX_MEMBERS];
};

#if ANI_OPND_FP16X2
__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// Four 8 x 8 matrices of 16-bit values into R: register j of lane l is row l / 4, columns 2 (l % 4) and 2 (l % 4) + 1
// of matrix j (the layout of an 8-column chunk of the wgmma accumulator), and lanes 8j .. 8j + 7 give the shared-window
// addresses of the eight 16-byte rows of matrix j.
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]),
               "r"(r[2]), "r"(r[3])
               : "memory");
}
// bulk copy shared -> global, tracked by this thread's bulk async-groups
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// this thread's bulk copies have finished reading their shared-memory source
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// this thread's bulk copies are complete: their writes are visible to this thread
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// D[64 x N] += A[64 x 16] * B[N x 16]^T for the N = 32, 64, 96 or 128 B rows of one ring slot (fp32 accumulate, both
// operands from shared memory).  The fragment is that of m64n64 products side by side: columns 0-63 in d0 (N = 32: its
// first 16 registers), columns 64-127 in d1.
#define ANI_RES_REGS16 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
#define ANI_RES_REGS32 ANI_RES_REGS16 ", %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define ANI_RES_REGS48 ANI_RES_REGS32 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
#define ANI_RES_REGS64 ANI_RES_REGS48 ", %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define ANI_RES_F8(d, i) \
  "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define ANI_RES_F16(d, i) ANI_RES_F8(d, i), ANI_RES_F8(d, i + 8)
#define ANI_RES_F32(d) ANI_RES_F16(d, 0), ANI_RES_F16(d, 16)
template <int N>
__device__ __forceinline__ void wgmma_res(float (&d0)[32], float (&d1)[32], uint64_t da, uint64_t db);
#define ANI_RES_WGMMA(N, REGS, DESCS, ...)                                                                       \
  template <>                                                                                                    \
  __device__ __forceinline__ void wgmma_res<N>(float (&d0)[32], float (&d1)[32], uint64_t da, uint64_t db) {     \
    (void)d1;                                                                                                    \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"                                                \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." ANI_WGMMA_AB " {" REGS "}, " DESCS            \
                 ", p, 1, 1, 0, 0;\n\t}"                                                                         \
                 : __VA_ARGS__                                                                                   \
                 : "l"(da), "l"(db));                                                                            \
  }
ANI_RES_WGMMA(32, ANI_RES_REGS16, "%16, %17", ANI_RES_F16(d0, 0))
ANI_RES_WGMMA(64, ANI_RES_REGS32, "%32, %33", ANI_RES_F32(d0))
ANI_RES_WGMMA(96, ANI_RES_REGS48, "%48, %49", ANI_RES_F32(d0), ANI_RES_F16(d1, 0))
ANI_RES_WGMMA(128, ANI_RES_REGS64, "%64, %65", ANI_RES_F32(d0), ANI_RES_F32(d1))
#undef ANI_RES_WGMMA
#undef ANI_RES_F32
#undef ANI_RES_F16
#undef ANI_RES_F8
#undef ANI_RES_REGS64
#undef ANI_RES_REGS48
#undef ANI_RES_REGS32
#undef ANI_RES_REGS16

// One commit group: the three products of the 2 x fp16 split (smallest terms first) of every K-step of one K-block, A
// at sa and the N B rows of one ring slot at sb.  N is a compile-time width because ptxas closes every branch inside a
// group with its own wgmma group boundary: a run-time width there split the group into one group per K-step, so
// wgmma.wait_group 1 waited for all of them, and ptxas injected a warpgroup.arrive (C7519) before every run.
template <int N>
__device__ __forceinline__ void res_mma_group(float (&d0)[32], float (&d1)[32], uint32_t sa, uint32_t sb) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < TK / 16; ++k) {
    const uint32_t adv = 32u * k;  // 16 pieces = 32 B along the swizzle row
    uint64_t da[PARTS], db[PARTS];
#pragma unroll
    for (int pp = 0; pp < PARTS; ++pp) {
      da[pp] = make_desc(sa + pp * A_PART_BYTES + adv);
      db[pp] = make_desc(sb + pp * A_PART_BYTES + adv);
    }
    wgmma_res<N>(d0, d1, da[1], db[0]);
    wgmma_res<N>(d0, d1, da[0], db[1]);
    wgmma_res<N>(d0, d1, da[0], db[0]);
  }
  wgmma_commit();
}
template <int N>
using ResWidth = std::integral_constant<int, N>;

// chain c of the list: species in `order`, then row tile, then member (SLABS: the members of member_of only).
// false: past the end
template <bool SLABS>
__device__ __forceinline__ bool res_chain(const ResArgs& a, const int* first, int c, int& s, int& rt, int& m) {
  const int cm = SLABS ? a.n_chain_members : a.members;
  for (int i = 0; i < a.num_species; ++i) {
    const int t = a.order[i];
    const int n = (first[t + 1] - first[t]) * cm;
    if (c < n) {
      s = t;
      rt = first[t] + c / cm;
      m = SLABS ? a.member_of[c % cm] : c % cm;
      return true;
    }
    c -= n;
  }
  return false;
}

// The r-th chain of this CTA: round r of gridDim.x chains, every other round in reverse CTA order.  The list is sorted
// longest first, so a CTA that took one of the first (longest) chains of a round takes one of the last (shortest) of
// the next: with 2-3 chains per CTA (a GDB batch of 256: H, C, N, O) the busiest CTA gets H + N + O instead of H + C + O.
__device__ __forceinline__ int res_chain_id(int r) {
  return r * (int)gridDim.x + ((r & 1) ? (int)gridDim.x - 1 - (int)blockIdx.x : (int)blockIdx.x);
}

// K-blocks of the A operand and output columns of phase p (nblk < 0: every AEV block is live)
__device__ __forceinline__ void res_phase(const ResArgs& a, const ResSpecies& sp, int p, int nblk, int& nkb, int& n) {
  switch (p) {
    case 0: nkb = nblk >= 0 ? nblk : a.kbx; n = sp.h1; break;
    case 1: nkb = sp.h1 / TK; n = sp.h2; break;
    case 2: nkb = sp.h2 / TK; n = sp.h3; break;
    case 3: nkb = sp.h3 / TK; n = sp.h2; break;
    case 4: nkb = sp.h2 / TK; n = sp.h1; break;
    default: nkb = sp.h1 / TK; n = nblk >= 0 ? nblk * TK : a.ldx; break;
  }
}

// ---- epilogue of one consumer warpgroup and phase P: 64 rows x bn columns from the accumulator registers ----
// Same register -> (row, column) map as tile_epilogue (gemm_tc.cuh).
template <int P, int ACT, bool SLABS>
__device__ __forceinline__ void res_epilogue(const ResArgs& a, const ResSpecies& sp, int rt, int m, int n0, int bn,
                                             float (&acc)[4][32], uint32_t res, const int* blk, int nblk, int wg,
                                             int lane, int warp_in_wg, float& omax) {
  constexpr bool ACTV = P <= 1, HEAD = P == 2, DCELU = P == 3 || P == 4, PLAIN = P == 5, GELU = ACT == ACT_GELU;
  const CeluConst cc{a.alpha, 1.0f / a.alpha, 1.4426950408889634f / a.alpha};
  const int q = lane & 3;
  const int r0 = 64 * wg + 16 * warp_in_wg + (lane >> 2);  // rows r0 and r0 + 8 of the tile
  const float acc_scale = sp.acc_scale[P];
  const float out_scale = ACTV ? OPND_SCALE_VALUE : OPND_SCALE_GRAD;
  // the global copy of a1 / a2 that phases 4 / 3 read back for CELU' (bulk-copied from R after phases 0 / 1), or
  // GELU: d1 / d2, stored there by phases 0 / 1
  unsigned char* ct = nullptr;
  if (P == 4 || (GELU && P == 0)) ct = a.act1 + ((size_t)rt * a.kb1 + (size_t)(m * sp.h1) / TK) * A_BLOCK_BYTES;
  if (P == 3 || (GELU && P == 1)) ct = a.act2 + ((size_t)rt * a.kb2 + (size_t)(m * sp.h2) / TK) * A_BLOCK_BYTES;
  const float* bias = !GELU && P <= 2 ? sp.bias[P] + (size_t)m * (P == 0 ? sp.h1 : P == 1 ? sp.h2 : sp.h3) : nullptr;
  const float* w4 = HEAD ? sp.w4 + (size_t)m * sp.h3 : nullptr;
  float e_acc[2] = {0.f, 0.f}, seed[2] = {0.f, 0.f};
  bool row_valid[2] = {false, false};
  if (HEAD) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      row_valid[h] = a.row_atom[rt * TM + r0 + 8 * h] >= 0;
      seed[h] = row_valid[h] ? a.member_scale[m] : 0.f;
    }
  }
  const int ngroups = bn / 32;
  // stmatrix: lane l gives the address of row 8h + (l & 7) of this warp's 16 rows, chunk l >> 3 (piece 0, group 0)
  uint32_t st_off[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) st_off[h] = res + swz_off(64 * wg + 16 * warp_in_wg + 8 * h + (lane & 7), lane >> 3);
  // dCELU: the stored activation of the next (32-column group, row half) is loaded before the current one is computed.
  // The thread loads the words of its own fragment, word q of chunk j of its row: columns 8j + 2q and 8j + 2q + 1.
  // L2 only (.cg): the words were written there by the bulk copy, never through this SM's L1.
  uint32_t ybuf[2][PARTS][4];
  auto load_y = [&](int g, int h, uint32_t (&dst)[PARTS][4]) {
    const int row = r0 + 8 * h;
    const unsigned char* b = ct + (size_t)g * A_BLOCK_BYTES + 4 * q;
#pragma unroll
    for (int p = 0; p < PARTS; ++p)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        dst[p][j] = __ldcg(reinterpret_cast<const unsigned int*>(b + p * A_PART_BYTES + swz_off(row, j)));
  };
  if (DCELU) load_y(0, 0, ybuf[0]);
  // One loop iteration per 32-column group, NOT unrolled: the body is compiled once per phase instead of eight times.
  // Unrolled, the kernel was 23 k instructions and its epilogues took twice as long on the H100, most likely because
  // every epilogue ran from a cold instruction cache.  The group's 16 accumulator registers are selected into `ag`
  // first (static register names).
#pragma unroll 1
  for (int g = 0; g < ngroups; ++g) {
    float ag[16];
    switch (g) {
#define ANI_RES_PICK(G)                                                     \
  case G:                                                                   \
    _Pragma("unroll") for (int i = 0; i < 16; ++i) ag[i] = acc[(G) >> 1][((G) & 1) * 16 + i]; \
    break;
      ANI_RES_PICK(0) ANI_RES_PICK(1) ANI_RES_PICK(2) ANI_RES_PICK(3)
      ANI_RES_PICK(4) ANI_RES_PICK(5) ANI_RES_PICK(6)
      default: ANI_RES_PICK(7)
#undef ANI_RES_PICK
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + 8 * h;
      if (DCELU) {
        if (h == 0)
          load_y(g, 1, ybuf[1]);
        else if (g + 1 < ngroups)
          load_y(g + 1, 0, ybuf[0]);
      }
      uint32_t w[PARTS][4];
      float o[4][2], od[2];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = 32 * g + 8 * j + 2 * q;  // column inside the tile
        float2 b2 = make_float2(0.f, 0.f), w2 = make_float2(0.f, 0.f), y2 = make_float2(0.f, 0.f);
        if (!GELU && P <= 2) b2 = __ldg(reinterpret_cast<const float2*>(bias + col));
        if (HEAD) w2 = __ldg(reinterpret_cast<const float2*>(w4 + col));
        if (DCELU) {
          uint32_t pw[PARTS];
#pragma unroll
          for (int p = 0; p < PARTS; ++p) pw[p] = ybuf[h][p][j];
          y2 = join_pair(pw);
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float v = ag[4 * j + 2 * h + e] * acc_scale;
          const float bb = e ? b2.y : b2.x, ww = e ? w2.y : w2.x, yy = e ? y2.y : y2.x;
          if (GELU && ACTV) {
            float d;
            gelu_and_grad(v, v, d);
            od[e] = d * OPND_SCALE_VALUE;
          } else if (GELU && DCELU) {
            v *= yy * (1.0f / OPND_SCALE_VALUE);
          } else if (GELU && HEAD) {
            float av, d;
            gelu_and_grad(v, av, d);
            e_acc[h] = fmaf(av, ww, e_acc[h]);
            v = seed[h] * ww * d;
          } else if (ACTV) {
            v = celu(v + bb, cc);
          } else if (DCELU) {
            v *= dcelu_from_out(yy * (1.0f / OPND_SCALE_VALUE), cc);
          } else if (HEAD) {
            const float av = celu(v + bb, cc);
            e_acc[h] = fmaf(av, ww, e_acc[h]);
            v = seed[h] * ww * dcelu_from_out(av, cc);
          }
          if (!PLAIN) {
            v *= out_scale;
            omax = max_abs_nan(omax, v);
          }
          o[j][e] = v;
        }
        if (!PLAIN) {
          uint32_t pw[PARTS];
          split_pair(o[j][0], o[j][1], pw);
#pragma unroll
          for (int p = 0; p < PARTS; ++p) w[p][j] = pw[p];
        }
        if (GELU && ACTV) {  // word q of chunk j of the row: the word load_y reads back
          uint32_t pw[PARTS];
          split_pair(od[0], od[1], pw);
          unsigned char* b = ct + (size_t)g * A_BLOCK_BYTES + 4 * q + swz_off(row, j);
#pragma unroll
          for (int p = 0; p < PARTS; ++p) *reinterpret_cast<uint32_t*>(b + p * A_PART_BYTES) = pw[p];
        }
      }
      if (PLAIN) {
        float* dst_row = a.dx + (SLABS ? (size_t)m * (size_t)a.slab_stride : (size_t)0) + (size_t)(rt * TM + row) * a.ldx;
        // live column blocks map back to their place: group g of the tile is live block n0 / 32 + g
        const int col0 = nblk >= 0 ? blk[n0 / 32 + g] * 32 : n0 + g * 32;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float* dst = dst_row + col0 + 8 * j + 2 * q;
          if (!SLABS && a.members > 1)
            red_add_v2(dst, o[j][0], o[j][1]);
          else
            *reinterpret_cast<float2*>(dst) = make_float2(o[j][0], o[j][1]);
        }
      } else {
        // matrix j of the stmatrix is chunk j of the group: whole 16-byte rows, swizzled by the lane addresses
#pragma unroll
        for (int p = 0; p < PARTS; ++p) stmatrix_x4(st_off[h] + (uint32_t)g * A_BLOCK_BYTES + p * A_PART_BYTES, w[p]);
      }
    }
  }
  if (HEAD) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float e = e_acc[h];
      e += __shfl_xor_sync(ANI_FULL_MASK, e, 1);
      e += __shfl_xor_sync(ANI_FULL_MASK, e, 2);
      if (q == 0) a.e_member[(size_t)m * a.rows_cap + rt * TM + r0 + 8 * h] = row_valid[h] ? e + sp.b4[m] : 0.f;
    }
  }
}

// ---- the kernel: one persistent CTA per SM, chains res_chain_id(0), res_chain_id(1), ... ----
// ACT: the activation of the model (ACT_CELU / ACT_GELU).
// SLABS = false: every member's chains, phase 5 reduces the members into dx (ani_b200_mlp_step_resident).
// SLABS = true: the chains of F.member_of only, phase 5 stores each member's rows into its own slab
// (ani_b200_mlp_step_resident_members).
template <int ACT, bool SLABS>
__global__ void __launch_bounds__(THREADS, 1) k_mlp_resident(const __grid_constant__ ResArgs F) {
  extern __shared__ unsigned char smem_raw[];
  // 1024-byte aligned (swizzle groups are 8 rows x 64 B): R, then the ring
  unsigned char* res = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* ring = res + RES_BYTES;
  __shared__ int s_first[ANI_MAX_SPECIES + 1];
  __shared__ int s_blk[MAX_BLOCKS];
  __shared__ __align__(8) uint64_t full[RES_SLOTS], empty[RES_SLOTS];
  const int warp = __shfl_sync(ANI_FULL_MASK, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int nblk = F.blocks ? min(F.blocks[0], MAX_BLOCKS) : -1;
  if (threadIdx.x <= F.num_species) s_first[threadIdx.x] = F.layout_info[4 + threadIdx.x];
  if ((int)threadIdx.x < nblk) s_blk[threadIdx.x] = F.blocks[1 + threadIdx.x];
  if (threadIdx.x == 32) {
    for (int i = 0; i < RES_SLOTS; ++i) {
      mbar_init(&full[i], 1);                     // the expect_tx arrival of the producer lane (+ the bytes)
      mbar_init(&empty[i], NUM_CONSUMER_WARPS);   // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  int s, rt, m;
  if (warp < 4) {
    setmaxnreg_dec<PROD_REGS>();
    if (warp != PROD_WARP) return;
    // ================================ producer (TMA) ================================
    uint32_t u = 0;  // ring slots handed out so far: slot u % RES_SLOTS, use u / RES_SLOTS of that slot
    for (int r = 0; res_chain<SLABS>(F, s_first, res_chain_id(r), s, rt, m); ++r) {
      const ResSpecies& sp = F.sp[s];
      for (int p = 0; p < RES_PHASES; ++p) {
        int nkb, n;
        res_phase(F, sp, p, nblk, nkb, n);
        // K-blocks of the stored B operand; phase 5 (W1^T of all members) starts member m at K-block m * h1 / 32
        const int nkb_all = p == 0 ? F.kbx : p == 5 ? F.members * sp.h1 / TK : nkb;
        const int kb_boff = p == 5 ? m * sp.h1 / TK : 0;
        const unsigned char* Bm = sp.B[p] + (p == 5 ? (size_t)0 : (size_t)m * n * nkb_all * (PARTS * ROW_BYTES));
        // phase 5 without the compact operand: lane -> (live block, piece) of a gathered 2 KB copy
        const bool gather = p == 5 && nblk >= 0 && !F.b_compact;
        for (int n0 = 0; n0 < n; n0 += TN_MAX) {
          const int bn = min(TN_MAX, n - n0);
          // slots of one K-block: the x block (phase 0), then one per 128 rows of B
          const int nh = (bn + RES_HALF - 1) / RES_HALF, a_sl = p == 0 ? 1 : 0;
          const int gq = lane / PARTS, gpart = lane % PARTS;
          const bool g_active = gather && lane < PARTS * (bn / 32);
          size_t g_src = 0;
          int g_bns = 0;
          if (g_active) {
            const int row0 = s_blk[n0 / 32 + gq] * 32, n0s = row0 / TN_MAX * TN_MAX;
            g_bns = min(TN_MAX, F.ldx - n0s);
            g_src = (size_t)n0s * nkb_all * (PARTS * ROW_BYTES) + (size_t)(row0 - n0s) * ROW_BYTES +
                    (size_t)gpart * g_bns * ROW_BYTES;
          }
          for (int kb = 0; kb < nkb; ++kb) {
            const int kbi = p == 0 && nblk >= 0 ? s_blk[kb] : kb;
            const int kbb = kbi + kb_boff;
            // B K-block in global memory: [p1 bn x 64 B | p2 bn x 64 B]
            const unsigned char* bsrc = Bm + ((size_t)n0 * nkb_all + (size_t)kbb * bn) * (PARTS * ROW_BYTES);
            // each slot is filled as soon as it is free: the consumers release a K-block's slots at different times
            for (int j = 0; j < a_sl + nh; ++j) {
              const int sl = (u + j) % RES_SLOTS;
              mbar_wait(&empty[sl], (((u + j) / RES_SLOTS) & 1) ^ 1);
              if (lane == 0) {
                if (j < a_sl) {
                  mbar_arrive_expect_tx(&full[sl], A_BLOCK_BYTES);
                  bulk_g2s(ring + sl * RES_SLOT_BYTES, F.x + ((size_t)rt * F.kbx + kbi) * A_BLOCK_BYTES, A_BLOCK_BYTES,
                           &full[sl]);
                } else {
                  const int h = j - a_sl;
                  const uint32_t rows = (uint32_t)min(RES_HALF, bn - h * RES_HALF);
                  mbar_arrive_expect_tx(&full[sl], PARTS * rows * ROW_BYTES);
                  if (!gather)
#pragma unroll
                    for (int pp = 0; pp < PARTS; ++pp)
                      bulk_g2s(ring + sl * RES_SLOT_BYTES + pp * A_PART_BYTES,
                               bsrc + ((size_t)pp * bn + h * RES_HALF) * ROW_BYTES, rows * ROW_BYTES, &full[sl]);
                }
              }
            }
            __syncwarp();
            if (g_active)
              bulk_g2s(ring + ((u + gq / 4) % RES_SLOTS) * RES_SLOT_BYTES + gpart * A_PART_BYTES +
                           (gq % 4) * 32 * ROW_BYTES,
                       Bm + g_src + (size_t)kbb * g_bns * (PARTS * ROW_BYTES), 32 * ROW_BYTES,
                       &full[(u + gq / 4) % RES_SLOTS]);
            __syncwarp();
            u += a_sl + nh;
          }
        }
      }
    }
    return;
  }

  // ================================ consumers ================================
  setmaxnreg_inc<CONS_REGS>();
  const int wg = (warp >> 2) - 1, warp_in_wg = warp & 3;
  const uint32_t res_u32 = smem_u32(res), res_a = res_u32 + wg * (64 / 8) * GROUP_BYTES;  // this warpgroup's rows of R
  const bool copier = warp_in_wg == 0 && lane == 0;  // issues and waits for the warpgroup's bulk copies of a1 / a2
  uint32_t u = 0;    // ring slots consumed so far, in the producer's order
  float omax = 0.f;  // largest |scaled value| this thread handed to the half-precision split
  for (int r = 0; __shfl_sync(ANI_FULL_MASK, (int)res_chain<SLABS>(F, s_first, res_chain_id(r), s, rt, m), 0); ++r) {
    const ResSpecies& sp = F.sp[s];
#pragma unroll 1
    for (int p = 0; p < RES_PHASES; ++p) {
      int nkb_, n_;
      res_phase(F, sp, p, nblk, nkb_, n_);
      const int nkb = __shfl_sync(ANI_FULL_MASK, nkb_, 0), n = __shfl_sync(ANI_FULL_MASK, n_, 0);
      for (int n0 = 0; n0 < n; n0 += TN_MAX) {
        const int bn = min(TN_MAX, n - n0);
        const int a_sl = p == 0 ? 1 : 0, nslot = a_sl + (bn + RES_HALF - 1) / RES_HALF;
        float acc[4][32];
        // A K-block's products are two commit groups, one per B slot (the second only if W1 > 0).  Every slot goes back
        // to the producer as soon as the last group that reads it has retired: B rows 0-127 after group 1, the A slot
        // (phase 0) and B rows 128-255 after group 2.  One group stays queued behind the one retiring, so the tensor
        // pipe keeps its overlap while the ring keeps as many slots in flight as it can (the weight feed is bound by
        // L2 latency, DESIGN §4.1).  The two groups accumulate into different registers, so the sums are those of
        // one interleaved group.
        auto release = [&](uint32_t base, uint32_t mask) {
          if (lane == 0)
            for (int j = 0; j < 3; ++j)
              if (mask >> j & 1) mbar_arrive(&empty[(base + j) % RES_SLOTS]);
        };
        // W0 / W1: the B rows of the K-block's two slots, as wide as each wgmma of the slot (the 32-128 columns of the
        // remainder, so no MMA runs on padding)
        auto main_loop = [&](auto w0_, auto w1_) {
          constexpr int W0 = decltype(w0_)::value, W1 = decltype(w1_)::value;
          // zero only the W0 + W1 columns the instance accumulates and the epilogue reads (w columns of a 64-column
          // slice are its registers 0 .. w / 2 - 1): the others stay dead, where zeros would be copied into every one
          // of them at the exit of every instance
          auto zero = [&](float (&d)[32], int w) {
#pragma unroll
            for (int i = 0; i < 32; ++i)
              if (i < w / 2) d[i] = 0.f;
          };
          zero(acc[0], min(W0, 64));
          zero(acc[1], W0 - 64);
          zero(acc[2], min(W1, 64));
          zero(acc[3], W1 - 64);
          uint32_t prev = 0, held = 0;  // slots prev + j (bit j of held) still read by the previous K-block's last group
#pragma unroll 1
          for (int kb = 0; kb < nkb; ++kb) {
            for (int j = 0; j <= a_sl; ++j) mbar_wait(&full[(u + j) % RES_SLOTS], ((u + j) / RES_SLOTS) & 1);
            const uint32_t sa = p == 0 ? smem_u32(ring + (u % RES_SLOTS) * RES_SLOT_BYTES) + wg * (64 / 8) * GROUP_BYTES
                                       : res_a + kb * A_BLOCK_BYTES;
            res_mma_group<W0>(acc[0], acc[1], sa, smem_u32(ring + ((u + a_sl) % RES_SLOTS) * RES_SLOT_BYTES));
            wgmma_wait<1>();
            release(prev, held);
            if constexpr (W1 > 0) {
              mbar_wait(&full[(u + a_sl + 1) % RES_SLOTS], ((u + a_sl + 1) / RES_SLOTS) & 1);
              res_mma_group<W1>(acc[2], acc[3], sa, smem_u32(ring + ((u + a_sl + 1) % RES_SLOTS) * RES_SLOT_BYTES));
              wgmma_wait<1>();
              release(u, 1u << a_sl);
              held = ((1u << nslot) - 1) & ~(1u << a_sl);
            } else {
              held = (1u << nslot) - 1;
            }
            prev = u;
            u += nslot;
          }
          wgmma_wait<0>();
          release(prev, held);
        };
        switch (bn / 32) {  // W0 = min(bn, 128), W1 = bn - W0
          case 1: main_loop(ResWidth<32>{}, ResWidth<0>{}); break;
          case 2: main_loop(ResWidth<64>{}, ResWidth<0>{}); break;
          case 3: main_loop(ResWidth<96>{}, ResWidth<0>{}); break;
          case 4: main_loop(ResWidth<128>{}, ResWidth<0>{}); break;
          case 5: main_loop(ResWidth<128>{}, ResWidth<32>{}); break;
          case 6: main_loop(ResWidth<128>{}, ResWidth<64>{}); break;
          case 7: main_loop(ResWidth<128>{}, ResWidth<96>{}); break;
          default: main_loop(ResWidth<128>{}, ResWidth<128>{}); break;
        }
        // the copies of a1 / a2 have read R before the epilogues of phases 1 / 2 overwrite it, and have landed in
        // global memory before phase 3 reads act2 back (phase 4 reads act1, copied earlier)
        if (ACT == ACT_CELU && copier && (p == 1 || p == 2)) bulk_wait_read();
        if (ACT == ACT_CELU && copier && p == 3) bulk_wait();
        // every warp of the warpgroup is done reading R before any of them overwrites it
        if (p < 5) wg_bar(wg);
        switch (p) {
          case 0: res_epilogue<0, ACT, SLABS>(F, sp, rt, m, n0, bn, acc, res_u32, s_blk, nblk, wg, lane, warp_in_wg, omax); break;
          case 1: res_epilogue<1, ACT, SLABS>(F, sp, rt, m, n0, bn, acc, res_u32, s_blk, nblk, wg, lane, warp_in_wg, omax); break;
          case 2: res_epilogue<2, ACT, SLABS>(F, sp, rt, m, n0, bn, acc, res_u32, s_blk, nblk, wg, lane, warp_in_wg, omax); break;
          case 3: res_epilogue<3, ACT, SLABS>(F, sp, rt, m, n0, bn, acc, res_u32, s_blk, nblk, wg, lane, warp_in_wg, omax); break;
          case 4: res_epilogue<4, ACT, SLABS>(F, sp, rt, m, n0, bn, acc, res_u32, s_blk, nblk, wg, lane, warp_in_wg, omax); break;
          default: res_epilogue<5, ACT, SLABS>(F, sp, rt, m, n0, bn, acc, res_u32, s_blk, nblk, wg, lane, warp_in_wg, omax); break;
        }
        // this warpgroup's rows of the phase's output, visible to the next phase's wgmma
        if (p < 5) {
          fence_proxy_async_shared();
          wg_bar(wg);
        }
        // a1 / a2 to act1 / act2 for the dCELU epilogues: this warpgroup's 64 rows of each K-block and piece are 4 KB,
        // contiguous in R and in the tiled global operand
        if (ACT == ACT_CELU && copier && p <= 1) {
          unsigned char* ct = p == 0 ? F.act1 + ((size_t)rt * F.kb1 + (size_t)(m * sp.h1) / TK) * A_BLOCK_BYTES
                                     : F.act2 + ((size_t)rt * F.kb2 + (size_t)(m * sp.h2) / TK) * A_BLOCK_BYTES;
          const uint32_t off = wg * (64 / 8) * GROUP_BYTES;
          for (int g = 0; g < bn / TK; ++g)
#pragma unroll
            for (int pp = 0; pp < PARTS; ++pp) {
              const uint32_t o = g * A_BLOCK_BYTES + pp * A_PART_BYTES + off;
              bulk_s2g(ct + o, res_u32 + o, (64 / 8) * GROUP_BYTES);
            }
          bulk_commit();
        }
      }
    }
  }
  if (F.status && !(omax <= OPND_HALF_MAX)) atomicOr(F.status, ANI_STATUS_OPERAND_RANGE);
}
#endif  // ANI_OPND_FP16X2

}  // namespace tc
}  // namespace ani
