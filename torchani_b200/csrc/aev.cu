// Fused neighbour search + AEV forward, and AEV backward (forces), one warp per central atom.
//
// Forward (replaces neighbors.py:64-113,968-1002 + aev/_computer.py:274-350; the reference's
// GPU path is csrc/aev.cu K1-K9).  One per-atom feature tail (atom_features), two ways to fill it with the
// neighbours in species-major order:
//   * k_aev_forward_cta (the bucket-grid path): the AEV_FWD_WARPS consecutive atoms of a CTA share the
//     27-bucket neighbourhood, staged once per CTA in shared memory in species-major order; a warp
//     compacts its neighbours with one ballot per 32 candidates and gets the neighbour list and the
//     angular sub-list grouped by species for free.
//   * k_aev_forward (explicit neighbour rows handed in by the caller, and ANI_B200_AEV_LEGACY=1): every
//     warp gathers its own neighbours (the rows, or its candidate ranges in global memory) and regroups
//     them by species (group_by_species).
// The tail: radial sums in registers, per species pair every lane evaluates whole triples (32 angular
// features in registers) + one warp transpose-reduce.  No atomics in the forward pass.
//
// Backward (csrc/aev.cu K10/K11): recomputes the geometry from the stored neighbour words, copies the
// live blocks of the upstream gradient row with cp.async into a compact per-composition table, and
// evaluates dE/dr_j over UNORDERED pairs by rotation (row j handles (j, j + t) once and hands the
// partner's share over with one shuffle); only the final per-neighbour vectors go to global memory
// (fire-and-forget float reductions), optionally with the f.r virial (stress) of ase.py:164-168.
#include <stdlib.h>

#include "common.cuh"
#include "terms.cuh"

namespace ani {

// ---- TMA bulk copy global -> shared with mbarrier completion (staging of the bucket ranges) ----------
__device__ __forceinline__ uint32_t aev_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void aev_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(aev_smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void aev_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(aev_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void aev_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   aev_smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(aev_smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void aev_mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "AEV_WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra.uni AEV_WAIT_DONE;\n\t"
      "bra.uni AEV_WAIT_LOOP;\n\t"
      "AEV_WAIT_DONE:\n\t"
      "}" ::"r"(aev_smem_u32(bar)),
      "r"(parity)
      : "memory");
}

constexpr int AEV_WARPS = 4;  // warps (= central atoms) per CTA
#ifndef ANI_AEV_BWD_MIN_CTAS
#define ANI_AEV_BWD_MIN_CTAS 7  // register budget of the backward kernel: 7 CTAs (28 warps) per SM
#endif
// the member loop of k_aev_backward_members keeps more state live: its ANI-2x form (8 x 4 angular terms) spills at 7
// and 6 CTAs per SM (72, 80 registers), not at 5 (96); the 4 x 8 form needs one CTA fewer (128)
#ifndef ANI_AEV_BWD_MEMBERS_MIN_CTAS
#define ANI_AEV_BWD_MEMBERS_MIN_CTAS 5
#endif

struct NeighbourRange {
  int lo, hi, code;
};

// Explicit per-atom neighbour rows (compute_from_neighbors path): atom i owns entries
// start[i] .. start[i+1]-1, each with the neighbour's atom index and (dx, dy, dz, R) = r_j - r_i.
struct ExplicitNbrs {
  const int32_t* start;
  const int32_t* j;
  const float4* d;
};

// r^2 of a neighbour vector, written out: both forward kernels must round it the same way (nvcc's own contraction of
// dx * dx + dy * dy + dz * dz depends on the surrounding code)
__device__ __forceinline__ float norm2(float dx, float dy, float dz) { return fmaf(dz, dz, fmaf(dx, dx, dy * dy)); }

// bucket range + image code for offset (ox, oy, oz) around bucket (ix, iy, iz) of the sub-grid that starts at
// bucket `base` (bucket_coords); false if it does not exist (non-periodic boundary)
__device__ __forceinline__ bool neighbour_bucket(const ani_grid& g, const int32_t* __restrict__ bin_start, int base,
                                                 int ix, int iy, int iz, int ox, int oy, int oz,
                                                 NeighbourRange& r) {
  int j[3] = {ix + ox, iy + oy, iz + oz};
  int w[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    w[d] = 0;
    if (j[d] < 0) {
      w[d] = -1;
      j[d] += g.dims[d];
    } else if (j[d] >= g.dims[d]) {
      w[d] = 1;
      j[d] -= g.dims[d];
    }
  }
  if (!g.pbc && (w[0] | w[1] | w[2])) return false;
  int b = base + (j[0] * g.dims[1] + j[1]) * g.dims[2] + j[2];
  r.lo = bin_start[b];
  r.hi = bin_start[b + 1];
  r.code = (w[0] + 1) * 9 + (w[1] + 1) * 3 + (w[2] + 1);
  return true;
}

// per-warp shared memory carve-up (byte offsets), shared by forward and backward
struct WarpSmem {
  float4* nd;            // [cap] dx, dy, dz, R   (neighbour - centre; the forward gathers r^2 into .w)
  float* nfc;            // [cap] forward: fc(R; Rcr).  backward: unused
  int32_t* nj;           // [cap] neighbour word
  float* fgrad;          // [cap*3] backward only
  unsigned char* nsp;    // [cap] species
  unsigned char* aidx;   // [ANI_MAX_ANG] angular neighbours (index into nd), species-sorted
  float* afc;            // [ANI_MAX_ANG] fc(R; Rca)
  float* afcd;           // [ANI_MAX_ANG] d fc / dR (backward)
  int32_t* seg;          // [ANI_MAX_SPECIES + 1] species segments of aidx
  int32_t* seg_all;      // [ANI_MAX_SPECIES + 1] species segments of nd (forward)
  float* rad;            // forward: [2*RL] accumulators; backward: g_rad [RL] + g_ang [pairs][36]
};

__host__ __device__ inline size_t warp_smem_bytes(int cap, int rad_floats, bool backward) {
  size_t b = (size_t)cap * 16 + (size_t)cap * 4 + (size_t)cap * 4;
  if (backward) b += (size_t)cap * 12;
  b += (size_t)cap;                          // nsp
  b += ANI_MAX_ANG;                          // aidx
  b = (b + 15) / 16 * 16;
  b += (size_t)ANI_MAX_ANG * 4 * 2;          // afc, afcd
  b += 2 * 16 * 4;                           // seg, seg_all (padded)
  b += ((size_t)cap + 15) / 16 * 16;         // unused; the launch shapes, occupancies and TMA staging capacity
                                             // of the kernels were tuned with these bytes in place
  b += (size_t)rad_floats * 4;
  return (b + 15) / 16 * 16;
}

__device__ __forceinline__ WarpSmem carve(unsigned char* base, int cap, bool backward) {
  WarpSmem s;
  unsigned char* p = base;
  s.nd = reinterpret_cast<float4*>(p);
  p += (size_t)cap * 16;
  s.nfc = reinterpret_cast<float*>(p);
  p += (size_t)cap * 4;
  s.nj = reinterpret_cast<int32_t*>(p);
  p += (size_t)cap * 4;
  s.fgrad = reinterpret_cast<float*>(p);
  if (backward) p += (size_t)cap * 12;
  s.nsp = p;
  p += cap;
  s.aidx = p;
  p += ANI_MAX_ANG;
  p = base + ((size_t)(p - base) + 15) / 16 * 16;
  s.afc = reinterpret_cast<float*>(p);
  p += ANI_MAX_ANG * 4;
  s.afcd = reinterpret_cast<float*>(p);
  p += ANI_MAX_ANG * 4;
  s.seg = reinterpret_cast<int32_t*>(p);
  p += 16 * 4;
  s.seg_all = reinterpret_cast<int32_t*>(p);
  p += 16 * 4;
  p += ((size_t)cap + 15) / 16 * 16;
  s.rad = reinterpret_cast<float*>(p);
  return s;
}

// Order-preserving compaction of the neighbours within Rca (backward pass): the pair rotation there looks the
// species of both partners up per pair and needs neither species segments nor a species-sorted list: one ballot per
// 32 neighbours, no counting sort.  Fills aidx/afc/afcd, returns the count (clamped to ANI_MAX_ANG).
__device__ __forceinline__ int compact_angular_list(const ani_aev_params& P, const WarpSmem& s, int cnt, int lane,
                                                    int32_t* status) {
  const unsigned lt = (1u << lane) - 1u;
  int total = 0;
  for (int base = 0; base < cnt; base += 32) {
    const int n = base + lane;
    const float R = n < cnt ? s.nd[n].w : 3.0e38f;
    const bool keep = R <= P.rca;
    const unsigned m = __ballot_sync(ANI_FULL_MASK, keep);
    const int pos = total + __popc(m & lt);
    if (keep && pos < ANI_MAX_ANG) {
      float f, df;
      cutoff_value_grad(R, P.rca, P.cutoff_kind, f, df);
      s.aidx[pos] = (unsigned char)n;
      s.afc[pos] = f;
      s.afcd[pos] = df;
    }
    total += __popc(m);
  }
  if (total > ANI_MAX_ANG) {
    if (lane == 0) atomicOr(status, ANI_STATUS_ANG_OVERFLOW);
    total = ANI_MAX_ANG;
  }
  __syncwarp();
  return total;
}

// one level of transpose_reduce32: lanes l and l ^ HALF swap halves of acc[0, 2 HALF) and each keeps a sum
template <int HALF>
__device__ __forceinline__ void transpose_level(float (&acc)[32], int lane) {
  const bool up = (lane & HALF) != 0;
#pragma unroll
  for (int i = 0; i < HALF; ++i) {
    float send = up ? acc[i] : acc[i + HALF];
    float keep = up ? acc[i + HALF] : acc[i];
    acc[i] = keep + __shfl_xor_sync(ANI_FULL_MASK, send, HALF);
  }
}

// sum acc[f] over the 32 lanes; lane l returns the total of feature l (31 shuffles).  The levels are template
// instances so that every index into acc is a constant: written as a loop over `half`, nvcc kept it rolled, which put
// the 32 accumulators on the stack and cost a local-memory store and load around every shuffle.
__device__ __forceinline__ float transpose_reduce32(float (&acc)[32], int lane) {
  transpose_level<16>(acc, lane);
  transpose_level<8>(acc, lane);
  transpose_level<4>(acc, lane);
  transpose_level<2>(acc, lane);
  transpose_level<1>(acc, lane);
  return acc[0];
}

// ---------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------
#ifndef ANI_AEV_CAND_CAP
#define ANI_AEV_CAND_CAP 768
#endif
#ifndef ANI_AEV_FWD_MIN_CTAS
#define ANI_AEV_FWD_MIN_CTAS 6
#endif
constexpr int CAND_CAP = ANI_AEV_CAND_CAP;
#ifndef ANI_AEV_FWD_WARPS
#define ANI_AEV_FWD_WARPS 4
#endif
constexpr int AEV_FWD_WARPS = ANI_AEV_FWD_WARPS;  // atoms (= warps) per CTA of the staged forward kernel
constexpr int NRANGE = 27;
constexpr int T2O_CAP = 1024;

// ---- opt-in phase trace (build variant "aevtrace": -DANI_AEV_FWD_TRACE=1; tools/aev_forward_trace.py) --------------
// One record of 16 int64 per atom (index i - lo), written by its warp: clock64 cycles spent in each phase (the staging
// phases include the CTA barriers that close them), %globaltimer and clock64 at the warp's start and end, the SM.
// Absent from the default build.
#ifndef ANI_AEV_FWD_TRACE
#define ANI_AEV_FWD_TRACE 0
#endif
enum AevTracePhase { TR_RANGES, TR_COUNT, TR_PLACE, TR_COMPACT, TR_LIST, TR_RADIAL, TR_ANGULAR, TR_PHASES };
#if ANI_AEV_FWD_TRACE
__device__ long long* g_aev_fwd_trace;
struct AevTrace {
  long long acc[TR_PHASES];
  long long t, gt0, ck0;
  __device__ __forceinline__ static long long clk() {
    long long v;
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(v));
    return v;
  }
  __device__ __forceinline__ static long long gtime() {
    long long v;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(v));
    return v;
  }
  __device__ __forceinline__ void start() {
#pragma unroll
    for (int k = 0; k < TR_PHASES; ++k) acc[k] = 0;
    gt0 = gtime();
    ck0 = t = clk();
  }
  __device__ __forceinline__ void mark(int ph) {
    const long long c = clk();
    acc[ph] += c - t;
    t = c;
  }
  __device__ __forceinline__ void write(size_t rec, int lane) {
    if (lane != 0 || !g_aev_fwd_trace) return;
    long long* r = g_aev_fwd_trace + rec * 16;
#pragma unroll
    for (int k = 0; k < TR_PHASES; ++k) r[k] = acc[k];
    unsigned sm;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
    r[8] = gt0;
    r[9] = gtime();
    r[10] = ck0;
    r[11] = clk();
    r[12] = sm;
  }
};
#else
struct AevTrace {
  __device__ __forceinline__ void start() {}
  __device__ __forceinline__ void mark(int) {}
  __device__ __forceinline__ void write(size_t, int) {}
};
#endif

// Candidate range o (0 .. 26; o = 9 (ox + 1) + 3 (oy + 1) + (oz + 1)) of bucket b: atoms lo .. hi - 1 of the
// bucket-sorted arrays, their image code and shift, and (range table only) the id of the neighbouring bucket, which
// addresses its per-bucket species offsets.  Mode 1 (bucket == conformer) has range 13 alone.  The range table, when
// given, holds the records; otherwise they are computed, the shift from the grid or, with LAT (grid mode 3), from the
// lattice of the bucket's conformer.  A range that does not exist (non-periodic boundary) is empty with code 13.
struct RangeRecord {
  int lo, hi, code, bucket;
  float3 shift;
};

template <bool LAT>
__device__ __forceinline__ RangeRecord bucket_range(const ani_grid& g, const int32_t* __restrict__ bin_start,
                                                   const float4* __restrict__ ranges, const float* __restrict__ lattice,
                                                   int b, int o) {
  RangeRecord r{0, 0, 13, b, make_float3(0.f, 0.f, 0.f)};
  if (g.mode == 1) {
    if (o == 13) {
      r.lo = bin_start[b];
      r.hi = bin_start[b + 1];
    }
  } else if (ranges) {
    const float4 r0 = ranges[2 * ((size_t)b * NRANGE + o)];
    const float4 r1 = ranges[2 * ((size_t)b * NRANGE + o) + 1];
    r.lo = __float_as_int(r0.x);
    r.hi = __float_as_int(r0.y);
    r.code = __float_as_int(r0.z);
    r.bucket = __float_as_int(r0.w);
    r.shift = make_float3(r1.x, r1.y, r1.z);
  } else {
    int ix, iy, iz;
    const int base = bucket_coords(g, b, ix, iy, iz);
    NeighbourRange n;
    if (neighbour_bucket(g, bin_start, base, ix, iy, iz, o / 9 - 1, (o / 3) % 3 - 1, o % 3 - 1, n)) {
      r.lo = n.lo;
      r.hi = n.hi;
      r.code = n.code;
      if (n.code != 13)
        r.shift = LAT ? image_shift(lattice, base / (g.dims[0] * g.dims[1] * g.dims[2]), n.code)
                      : image_shift(g, n.code);
    }
  }
  return r;
}

// A lane's stores into one AEV row: plain row-major (layout 0), or the tiled operand layout (16-bit pieces) the GEMM
// consumes.  vmax is the largest scaled feature the lane wrote, for the operand range check of the fp16 pieces.
struct FeatureWriter {
  float* aev;
  int row, ldx, kblocks, layout;
  float vmax;
  __device__ __forceinline__ void operator()(int col, float v) {
    if (layout == 0) {
      aev[(size_t)row * ldx + col] = v;
    } else {
      unsigned char* dst = reinterpret_cast<unsigned char*>(aev) + opnd_offset(row, col, kblocks);
      unsigned short pc[OPND_PARTS];
      v *= OPND_SCALE_VALUE;
      vmax = fmaxf(vmax, v);  // AEV features are >= 0
      opnd_split(v, pc);
#pragma unroll
      for (int k = 0; k < OPND_PARTS; ++k) *reinterpret_cast<unsigned short*>(dst + k * OPND_PART_BYTES) = pc[k];
    }
  }
};

// The features of atom i from its neighbourhood in the warp's shared memory: the per-atom tail of both forward
// kernels.  Input: nd[n] = (dx, dy, dz, r^2) of the neighbours within Rcr in species-major order, nj[n] their
// words, seg_all the species segments of that list, aidx the angular sub-list (r^2 <= Rca^2, indices into nd) and
// seg its species segments; cnt and cnt_a unclamped (an overflow sets its status bit).  Writes nbr_cnt / nbr_list
// (when given) and the AEV row of atom i.
template <int NA, int NZ>
__device__ __forceinline__ void atom_features(const ani_aev_params& P, const WarpSmem& s, int i, int cnt, int cnt_a,
                                              const int32_t* __restrict__ species_mask,
                                              const int32_t* __restrict__ row_of, float* __restrict__ aev, int ldx,
                                              int layout, int32_t* __restrict__ nbr_cnt,
                                              int32_t* __restrict__ nbr_list, int cap, int32_t* __restrict__ status,
                                              AevTrace& tr) {
  const int lane = threadIdx.x & 31;
  const int S = P.num_species;
  const int nR = P.n_shf_r;
  const int RL = S * nR;
  if (cnt > cap) {
    if (lane == 0) atomicOr(status, ANI_STATUS_NBR_OVERFLOW);
    cnt = cap;
  }
  if (cnt_a > ANI_MAX_ANG) {
    if (lane == 0) atomicOr(status, ANI_STATUS_ANG_OVERFLOW);
    cnt_a = ANI_MAX_ANG;
  }
  __syncwarp();

  FeatureWriter store{aev, row_of[i], ldx, ldx >> 5, layout, 0.f};

  if (lane == 0 && nbr_cnt) nbr_cnt[i] = cnt;
  // per neighbour: (c R, fc(R)) with c = sqrt(eta_r log2 e), so that a Gaussian factor is
  // ex2(-(c R - c ShfR)^2); the neighbour words go to the list the backward kernel reads
  const float cr = sqrtf(P.eta_r * 1.4426950408889634f);
  if (nbr_list)
    for (int n = lane; n < cnt; n += 32) nbr_list[(size_t)i * cap + n] = s.nj[n];
  __syncwarp();
  // [cap] float2 over nfc and nj (adjacent, 8-byte aligned; the words were just copied out)
  float2* rf = reinterpret_cast<float2*>(s.nfc);
  for (int n = lane; n < cnt; n += 32) {
    const float R = sqrtf(s.nd[n].w);
    s.nd[n].w = R;
    rf[n] = make_float2(cr * R, cutoff_value(R, P.rcr, P.cutoff_kind));
  }
  __syncwarp();
  tr.mark(TR_LIST);

  // element pairs / elements that do not occur anywhere in the system are never read by the MLP:
  // skip them (species_mask[1] != 0: the composition changed since the last call -> write them once)
  const unsigned present = (species_mask && !species_mask[1]) ? (unsigned)species_mask[0] : 0xffffffffu;

  // ---- radial block: lane = (shift m, neighbour parity h); one species segment at a time, the
  //      (species, shift) sum lives in a register: no shared-memory accumulators, no atomics
  {
    const int lpn = (nR <= 16) ? 16 : 32;
    const int halves = 32 / lpn;
    const int m = lane % lpn, h = lane / lpn;
    const float cshf = cr * P.shf_r[m < nR ? m : 0];
    for (int sp = 0; sp < S; ++sp) {
      if (!((present >> sp) & 1u)) continue;
      const int k1 = s.seg_all[sp + 1];
      float acc = 0.f;
#pragma unroll 2
      for (int k = s.seg_all[sp] + h; k < k1; k += halves) {
        const float2 v = rf[k];
        const float d = v.x - cshf;
        acc = fmaf(fast_exp2(-d * d), v.y, acc);
      }
      if (halves == 2) acc += __shfl_xor_sync(ANI_FULL_MASK, acc, 16);
      if (h == 0 && m < nR) store(sp * nR + m, 0.25f * acc);
    }
  }
  tr.mark(TR_RADIAL);

  // ---- angular block
  const int n_ang = cnt_a;
  for (int q = lane; q < n_ang; q += 32) s.afc[q] = cutoff_value(s.nd[s.aidx[q]].w, P.rca, P.cutoff_kind);
  __syncwarp();
  // f2[a] * w = ex2(-(ca rbar - ca ShfA)^2 + lg2 w),  f1[z] = (0.5 + c (cz/2) + s (sz/2))^zeta
  const float ca = sqrtf(P.eta_a * 1.4426950408889634f);
  float cshfA[NA], hcz[NZ], hsz[NZ];
#pragma unroll
  for (int a = 0; a < NA; ++a) cshfA[a] = ca * P.shf_a[a];
#pragma unroll
  for (int z = 0; z < NZ; ++z) {
    hcz[z] = 0.5f * P.cos_z[z];
    hsz[z] = 0.5f * P.sin_z[z];
  }
  // walk the set bits of the element mask: pairs (s1, s2 >= s1) of present elements only
  for (unsigned m1 = present & ((1u << S) - 1u); m1; m1 &= m1 - 1) {
    const int s1 = __ffs(m1) - 1;
    const int a0 = s.seg[s1], na = s.seg[s1 + 1] - a0;
    const int pbase = s1 * (2 * S - s1 + 1) / 2 - s1;  // pair_index(s1, s2) = pbase + s2
    for (unsigned m2 = m1; m2; m2 &= m2 - 1) {
      const int s2 = __ffs(m2) - 1;
      const int p = pbase + s2;
      const int b0 = s.seg[s2], nb = s.seg[s2 + 1] - b0;
      const int count = (s1 == s2) ? na * (na - 1) / 2 : na * nb;
      float out = 0.f;
      if (count > 0) {
        float acc[32];
#pragma unroll
        for (int f = 0; f < 32; ++f) acc[f] = 0.f;
        const float inv_nb = 1.0f / (float)nb;
        for (int q = lane; q < count; q += 32) {
          int ja, jb;
          if (s1 == s2) {
            // q-th pair (a < b) of the triangle: b = floor((1 + sqrt(1 + 8 q)) / 2), one fix-up each way
            int bb = (int)(0.5f + 0.5f * fast_sqrt(1.0f + 8.0f * (float)q));
            if (bb * (bb - 1) / 2 > q) --bb;
            if ((bb + 1) * bb / 2 <= q) ++bb;
            ja = a0 + q - bb * (bb - 1) / 2;
            jb = a0 + bb;
          } else {
            // q / nb for q < 2^13, nb <= 96: the float quotient of (q + 0.5) is never within rounding of an integer
            const int qa = (int)(((float)q + 0.5f) * inv_nb);
            ja = a0 + qa;
            jb = b0 + q - qa * nb;
          }
          const float4 dj = s.nd[s.aidx[ja]], dk = s.nd[s.aidx[jb]];
          const float lw = fast_log2(2.0f * s.afc[ja] * s.afc[jb]);  // -inf at the cutoff: every term 0
          const float dot = dj.x * dk.x + dj.y * dk.y + dj.z * dk.z;
          const float c = 0.95f * dot * fast_rcp(fmaxf(dj.w * dk.w, 1e-10f));
          const float sn = fast_sqrt(fmaxf(1.0f - c * c, 0.f));
          const float rbar = ca * 0.5f * (dj.w + dk.w);
          float f1[NZ];
#pragma unroll
          for (int z = 0; z < NZ; ++z) {
            const float base = fmaxf(fmaf(sn, hsz[z], fmaf(c, hcz[z], 0.5f)), 0.f);
            f1[z] = fast_exp2(P.zeta * fast_log2(base));  // base^zeta; base = 0 -> ex2(-inf) = 0
          }
#pragma unroll
          for (int a = 0; a < NA; ++a) {
            const float d = rbar - cshfA[a];
            const float f2 = fast_exp2(fmaf(-d, d, lw));
#pragma unroll
            for (int z = 0; z < NZ; ++z) acc[a * NZ + z] = fmaf(f1[z], f2, acc[a * NZ + z]);
          }
        }
        out = transpose_reduce32(acc, lane);
      }
      store(RL + (layout ? P.ang_pad : 0) + p * 32 + lane, out);
    }
  }
  if (ANI_OPND_FP16X2 && !(store.vmax <= OPND_HALF_MAX)) atomicOr(status, ANI_STATUS_OPERAND_RANGE);
  tr.mark(TR_ANGULAR);
}

// Stable regroup of a warp's first cnt neighbour rows (nd with r^2 in .w, nj, species nsp) into species-major order,
// then the angular sub-list with one ballot per 32 regrouped neighbours: the input of atom_features as the CTA
// kernel's compaction leaves it.  Each lane holds its rows in registers while they move (cnt <= nbr_cap <= 256); the
// running place of every species is kept in seg until the angular segments overwrite it.  Returns the number of
// angular neighbours (unclamped).
__device__ __forceinline__ int group_by_species(const ani_aev_params& P, const WarpSmem& s, int cnt) {
  constexpr int PER = 256 / 32;
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  int spv[PER];
  int seg_start[ANI_MAX_SPECIES + 1];
#pragma unroll
  for (int e = 0; e <= ANI_MAX_SPECIES; ++e) seg_start[e] = 0;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int n = k * 32 + lane;
    spv[k] = n < cnt ? (int)s.nsp[n] : -1;
    if (k * 32 < cnt) {
#pragma unroll
      for (int e = 0; e < ANI_MAX_SPECIES; ++e) seg_start[e + 1] += __popc(__ballot_sync(ANI_FULL_MASK, spv[k] == e));
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int e = 0; e < ANI_MAX_SPECIES; ++e) {
      seg_start[e + 1] += seg_start[e];
      s.seg[e] = seg_start[e];
      if (e <= P.num_species) s.seg_all[e] = seg_start[e];
    }
    if (P.num_species == ANI_MAX_SPECIES) s.seg_all[ANI_MAX_SPECIES] = seg_start[ANI_MAX_SPECIES];
  }
  __syncwarp();
  float4 d[PER];
  int w[PER], dst[PER];
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    dst[k] = -1;
    if (k * 32 < cnt) {
      const int e = spv[k];
      const bool placed = e >= 0 && e < ANI_MAX_SPECIES;
      const unsigned peers = __match_any_sync(ANI_FULL_MASK, e);  // the lanes of this species, in lane order
      if (placed) {
        dst[k] = s.seg[e] + __popc(peers & lt);
        d[k] = s.nd[k * 32 + lane];
        w[k] = s.nj[k * 32 + lane];
      }
      __syncwarp();
      if (placed && !(peers & lt)) s.seg[e] += __popc(peers);
      __syncwarp();
    }
  }
#pragma unroll
  for (int k = 0; k < PER; ++k)
    if (dst[k] >= 0) {
      s.nd[dst[k]] = d[k];
      s.nj[dst[k]] = w[k];
    }
  __syncwarp();
  // the angular sub-list: one ballot per 32 neighbours of the regrouped list; lane e < S counts the angular neighbours
  // before the end of species segment e, the boundary seg[e + 1]
  const float rca2 = P.rca * P.rca;
  const int end = s.seg_all[P.num_species];
  const int seg_end = lane < P.num_species ? s.seg_all[lane + 1] : 0;
  int cnt_a = 0, below = 0;
  for (int base = 0; base < end; base += 32) {
    const int n = base + lane;
    const bool keep_a = n < end && s.nd[n].w <= rca2;
    const unsigned ma = __ballot_sync(ANI_FULL_MASK, keep_a);
    const int pa = cnt_a + __popc(ma & lt);
    if (keep_a && pa < ANI_MAX_ANG) s.aidx[pa] = (unsigned char)n;
    cnt_a += __popc(ma);
    const int before = seg_end - base;
    below += __popc(ma & (before >= 32 ? 0xffffffffu : before <= 0 ? 0u : (1u << before) - 1u));
  }
  if (lane < P.num_species) s.seg[lane + 1] = min(below, ANI_MAX_ANG);
  if (lane == 0) s.seg[0] = 0;
  __syncwarp();
  return cnt_a;
}

// Warp-per-atom forward (explicit neighbour rows, and the bucket grid with ANI_B200_AEV_LEGACY=1): every warp gathers
// its own neighbours -- the caller's rows, or its bucket's 27 candidate ranges walked in global memory in range order
// -- regroups them by species and evaluates the shared tail.  On the bucket grid the neighbours come out in the order
// of k_aev_forward_cta (species, range, position), so both kernels give the same bits unless nbr_cap overflows.
// LAT (grid mode 3): image shifts in the lattice of the bucket's conformer (lattice table); the range table, when
// given, already holds them
template <int NA, int NZ, bool LAT = false>
__global__ void __launch_bounds__(AEV_WARPS * 32)
    k_aev_forward(const __grid_constant__ ani_aev_params P, const ani_grid* __restrict__ grid,
                  const int32_t* __restrict__ bin_start, const float4* __restrict__ spos,
                  const int32_t* __restrict__ sbin, const float4* __restrict__ ranges,
                  const int32_t* __restrict__ species_mask, const ExplicitNbrs ex, int lo, int hi,
                  const int32_t* __restrict__ row_of,
                  float* __restrict__ aev, int ldx, int layout, int32_t* __restrict__ nbr_cnt,
                  int32_t* __restrict__ nbr_list, int cap, int32_t* __restrict__ status, size_t warp_bytes,
                  const float* __restrict__ lattice) {
  static_assert(NA * NZ == 32, "one lane per angular feature");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  AevTrace tr;  // (the phase trace records k_aev_forward_cta only: nothing is written)
  tr.start();
  const ani_grid g = *grid;
  hi = min(hi, g.n_real);
  const int i = lo + blockIdx.x * AEV_WARPS + warp;
  if (i >= hi) return;
  const WarpSmem s = carve(smem_raw + warp * warp_bytes, cap, false);
  const float4 pi = spos[i];
  if (__float_as_int(pi.w) < 0) return;  // padding atom (only reachable with explicit neighbour rows)
  int cnt = 0;
  if (ex.start) {
    // neighbours handed in by the caller (already screened to Rcr): copy the row
    const int e0 = ex.start[i];
    cnt = ex.start[i + 1] - e0;
    for (int n = lane; n < min(cnt, cap); n += 32) {
      const int j = ex.j[e0 + n];
      const float4 d = ex.d[e0 + n];
      s.nd[n] = make_float4(d.x, d.y, d.z, norm2(d.x, d.y, d.z));
      s.nj[n] = j | (13 << ANI_IMG_SHIFT);
      s.nsp[n] = (unsigned char)__float_as_int(spos[j].w);
    }
  } else {
    // lane o holds the record of candidate range o; the warp compacts the atoms within Rcr range after range
    const float rcr2 = P.rcr * P.rcr;
    const unsigned lt = (1u << lane) - 1u;
    RangeRecord r{};
    if (lane < NRANGE) r = bucket_range<LAT>(g, bin_start, ranges, lattice, sbin[i], lane);
    for (int o = 0; o < NRANGE; ++o) {
      const int rlo = __shfl_sync(ANI_FULL_MASK, r.lo, o), rhi = __shfl_sync(ANI_FULL_MASK, r.hi, o);
      if (rhi <= rlo) continue;
      const int code = __shfl_sync(ANI_FULL_MASK, r.code, o);
      const float shx = __shfl_sync(ANI_FULL_MASK, r.shift.x, o), shy = __shfl_sync(ANI_FULL_MASK, r.shift.y, o),
                  shz = __shfl_sync(ANI_FULL_MASK, r.shift.z, o);
      for (int base = rlo; base < rhi; base += 32) {
        const int c = base + lane;
        const bool valid = c < rhi;
        const float4 p = valid ? spos[c] : pi;
        const float dx = (p.x + shx) - pi.x, dy = (p.y + shy) - pi.y, dz = (p.z + shz) - pi.z;
        const float r2 = norm2(dx, dy, dz);
        const bool keep = valid && r2 <= rcr2 && !(c == i && code == 13);
        const unsigned m = __ballot_sync(ANI_FULL_MASK, keep);
        const int pos = cnt + __popc(m & lt);
        if (keep && pos < cap) {
          s.nd[pos] = make_float4(dx, dy, dz, r2);
          s.nj[pos] = c | (code << ANI_IMG_SHIFT);
          s.nsp[pos] = (unsigned char)__float_as_int(p.w);
        }
        cnt += __popc(m);
      }
    }
  }
  __syncwarp();
  const int cnt_a = group_by_species(P, s, min(cnt, cap));
  atom_features<NA, NZ>(P, s, i, cnt, cnt_a, species_mask, row_of, aev, ldx, layout, nbr_cnt, nbr_list, cap, status,
                        tr);
}

// ---------------------------------------------------------------------------------------
// forward, CTA-staged neighbourhood (the bucket-grid path)
//
// The AEV_WARPS consecutive (bucket-sorted) atoms of a CTA almost always share one bucket, so the
// candidates of its 27 neighbouring buckets are staged ONCE per CTA in shared memory -- shifted by
// their lattice image and ordered species-major (the buckets are species-sorted, so the place of
// every candidate follows from a 27 x S table of counts) -- instead of every warp walking the 27
// ranges in global memory.  A warp then compacts its neighbours with one ballot per 32 candidates,
// species segment by species segment: the neighbour list and the angular sub-list come out
// grouped by species, ready for atom_features.
// CTAs that straddle a bucket boundary run one staging phase per distinct bucket; neighbourhoods
// larger than CAND_CAP candidates are staged in windows of the species-major order.
// ---------------------------------------------------------------------------------------
struct CtaStage {
  float4 cand[CAND_CAP];  // shifted position; .w = neighbour word (sorted index | image code << 26)
  float4 r_shift[NRANGE];
  int r_lo[NRANGE], r_code[NRANGE];
  int r_len[NRANGE];                           // candidates of every range
  int r_off[NRANGE + 1];                       // exclusive prefix of the range lengths
  int cnt[ANI_MAX_SPECIES][NRANGE];            // candidates per (species, range)
  int off[ANI_MAX_SPECIES * NRANGE + 1];       // exclusive prefix of cnt in species-major order
  int adj[ANI_MAX_SPECIES][NRANGE];            // off[s][o] - (candidates of lower species in range o)
  int wbin[AEV_FWD_WARPS];
  unsigned char t2o[T2O_CAP];                  // range of the t-th candidate (range-major numbering)
  unsigned long long tma_bar;                  // mbarrier of the TMA bulk copies that stage the bucket ranges
};

template <int NA, int NZ, bool TMA_STAGE = false, bool LAT = false>
__global__ void __launch_bounds__(AEV_FWD_WARPS * 32, ANI_AEV_FWD_MIN_CTAS)
    k_aev_forward_cta(const __grid_constant__ ani_aev_params P, const ani_grid* __restrict__ grid,
                      const int32_t* __restrict__ bin_start, const float4* __restrict__ spos,
                      const int32_t* __restrict__ sbin, const float4* __restrict__ ranges,
                      const int32_t* __restrict__ species_mask, int lo, int hi, const int32_t* __restrict__ row_of,
                      float* __restrict__ aev, int ldx, int layout, int32_t* __restrict__ nbr_cnt,
                      int32_t* __restrict__ nbr_list, int cap, int32_t* __restrict__ status, size_t warp_bytes,
                      int tma_stage, const int32_t* __restrict__ bss, const float* __restrict__ lattice) {
  static_assert(NA * NZ == 32, "one lane per angular feature");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ CtaStage C;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  AevTrace tr;
  tr.start();
  const ani_grid g = *grid;
  hi = min(hi, g.n_real);
  const int i = lo + blockIdx.x * AEV_FWD_WARPS + warp;
  const bool has = i < hi;  // warps without an atom still help with the staging
  const WarpSmem s = carve(smem_raw + warp * warp_bytes, cap, false);
  const int S = P.num_species;
  float4 pi = make_float4(0.f, 0.f, 0.f, 0.f);
  int myb = 0x7fffffff;
  if (has) {
    pi = spos[i];
    myb = sbin[i];
  }
  if (lane == 0) C.wbin[warp] = myb;
  if (TMA_STAGE && tid == 0) aev_mbar_init(reinterpret_cast<uint64_t*>(&C.tma_bar), 1);
  __syncthreads();

  // ---- 1. neighbours within Rcr (and the sub-list within Rca), species segment by species segment
  const float rcr2 = P.rcr * P.rcr, rca2 = P.rca * P.rca;
  const unsigned lt = (1u << lane) - 1u;
  int cnt = 0, cnt_a = 0;
  // TMA staging area: the per-warp arrays of the dynamic shared memory are not in use before the first compaction,
  // so the raw candidates of the FIRST bucket of the CTA (the only one for most CTAs) land there, range after range,
  // by cp.async.bulk -- the two staging passes below then read shared memory instead of global memory
  float4* raw = reinterpret_cast<float4*>(smem_raw);
  const int raw_cap = (int)min((size_t)CAND_CAP, (AEV_FWD_WARPS * warp_bytes) / sizeof(float4));
  uint32_t tma_parity = 0;
  int prev = -1, first_bucket = -1;
  const bool use_bss = bss != nullptr;
  while (true) {
    int cur = 0x7fffffff;
#pragma unroll
    for (int w = 0; w < AEV_FWD_WARPS; ++w) {
      const int b = C.wbin[w];
      if (b > prev && b < cur) cur = b;
    }
    if (cur == 0x7fffffff) break;
    if (prev == -1) first_bucket = cur;
    prev = cur;
    __syncthreads();  // every warp has chosen `cur`; the tables of the previous phase may be rewritten
    // (a) the 27 candidate ranges of bucket `cur`
    if (tid < NRANGE) {
      const RangeRecord r = bucket_range<LAT>(g, bin_start, ranges, lattice, cur, tid);
      C.r_lo[tid] = r.lo;
      C.r_code[tid] = r.code;
      C.r_shift[tid] = make_float4(r.shift.x, r.shift.y, r.shift.z, 0.f);
      const int len = max(r.hi - r.lo, 0);
      C.r_len[tid] = len;
      if (use_bss) {
        // candidates per (species, range) straight from the per-bucket species offsets of the preparation kernel
        // (buckets are species-sorted): no counting pass over the candidates, no shared-memory atomics
        int off8[ANI_MAX_SPECIES + 1];
        if (len > 0) {
          const int4 q0 = reinterpret_cast<const int4*>(bss)[2 * (size_t)r.bucket], q1 = reinterpret_cast<const int4*>(bss)[2 * (size_t)r.bucket + 1];
          off8[0] = q0.x; off8[1] = q0.y; off8[2] = q0.z; off8[3] = q0.w;
          off8[4] = q1.x; off8[5] = q1.y; off8[6] = q1.z; off8[7] = q1.w;
          off8[ANI_MAX_SPECIES] = len;
        } else {
#pragma unroll
          for (int k = 0; k <= ANI_MAX_SPECIES; ++k) off8[k] = 0;
        }
#pragma unroll
        for (int k = 0; k < ANI_MAX_SPECIES; ++k) C.cnt[k][tid] = off8[k + 1] - off8[k];
      }
    }
    if (!use_bss)
      for (int q = tid; q < ANI_MAX_SPECIES * NRANGE; q += AEV_FWD_WARPS * 32) (&C.cnt[0][0])[q] = 0;
    __syncthreads();
    // inclusive scan of the 27 lengths (lane o holds range o).  With the bss table EVERY warp computes the (identical)
    // prefixes itself: no warp idles at a CTA barrier while another one scans
    if (use_bss || warp == 0) {
      int v = lane < NRANGE ? C.r_len[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(ANI_FULL_MASK, v, o);
        if (lane >= o) v += y;
      }
      if (lane < NRANGE) C.r_off[lane + 1] = v;
      if (lane == 0) C.r_off[0] = 0;
      __syncwarp();
    }
    if (!use_bss) __syncthreads();
    tr.mark(TR_RANGES);
    const int T = C.r_off[NRANGE];
    // first bucket of the CTA, neighbourhood fits: one TMA bulk copy per non-empty range (contiguous float4 runs of
    // the bucket-sorted position array), all completing on one mbarrier
    const bool staged = TMA_STAGE && tma_stage && prev == first_bucket && T > 0 && T <= raw_cap;
    if (staged) {
      if (tid == 0) aev_mbar_expect_tx(reinterpret_cast<uint64_t*>(&C.tma_bar), (uint32_t)T * 16u);
      if (tid < NRANGE) {
        const int len = C.r_off[tid + 1] - C.r_off[tid];
        if (len > 0)
          aev_bulk_g2s(raw + C.r_off[tid], spos + C.r_lo[tid], (uint32_t)len * 16u, reinterpret_cast<uint64_t*>(&C.tma_bar));
      }
      aev_mbar_wait(reinterpret_cast<uint64_t*>(&C.tma_bar), tma_parity);
      tma_parity ^= 1u;
    }
    // flat (range-major) candidate number -> range: branch-free binary search over the prefix
    auto find_range = [&](int t) {
      int o = 0;
#pragma unroll
      for (int step = 16; step >= 1; step >>= 1)
        if (o + step < NRANGE && C.r_off[o + step] <= t) o += step;
      return o;
    };
    // (b) candidates per (species, range); the range of every candidate is remembered for (c)
    // (four candidates per thread and round: the global loads are issued together)
    constexpr int NT = AEV_FWD_WARPS * 32, BATCH = 4;
    for (int t0 = tid; t0 < T && !use_bss; t0 += NT * BATCH) {
      int oo[BATCH], spv[BATCH];
#pragma unroll
      for (int j = 0; j < BATCH; ++j) {
        const int t = t0 + j * NT;
        oo[j] = -1;
        if (t < T) {
          const int o = find_range(t);
          oo[j] = o;
          if (t < T2O_CAP) C.t2o[t] = (unsigned char)o;
          spv[j] = __float_as_int(staged ? raw[t].w : spos[C.r_lo[o] + (t - C.r_off[o])].w);
        }
      }
#pragma unroll
      for (int j = 0; j < BATCH; ++j)
        if (oo[j] >= 0) atomicAdd(&C.cnt[spv[j]][oo[j]], 1);
    }
    if (!use_bss) __syncthreads();
    if (use_bss || warp == 0) {
      // exclusive prefix over q = species * 27 + range: 7 consecutive entries per lane
      constexpr int PER = (ANI_MAX_SPECIES * NRANGE + 31) / 32;
      int loc[PER];
      int sum = 0;
#pragma unroll
      for (int k = 0; k < PER; ++k) {
        const int q = lane * PER + k;
        loc[k] = q < ANI_MAX_SPECIES * NRANGE ? (&C.cnt[0][0])[q] : 0;
        sum += loc[k];
      }
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(ANI_FULL_MASK, incl, o);
        if (lane >= o) incl += y;
      }
      int run = incl - sum;
#pragma unroll
      for (int k = 0; k < PER; ++k) {
        const int q = lane * PER + k;
        if (q <= ANI_MAX_SPECIES * NRANGE) C.off[q] = run;
        run += loc[k];
      }
      __syncwarp();
      // place of a candidate = adj[species][range] + its offset inside the (species-sorted) range
      if (lane < NRANGE) {
        int lower = 0;
#pragma unroll
        for (int sp = 0; sp < ANI_MAX_SPECIES; ++sp) {
          C.adj[sp][lane] = C.off[sp * NRANGE + lane] - lower;
          lower += C.cnt[sp][lane];
        }
      }
      __syncwarp();
    }
    if (!use_bss) __syncthreads();
    tr.mark(TR_COUNT);
    const bool mine = has && myb == cur;
    for (int F0 = 0; F0 < T; F0 += CAND_CAP) {
      // (c) place the candidates whose species-major position falls into this window
      for (int t0 = tid; t0 < T; t0 += NT * BATCH) {
        int oo[BATCH], cc[BATCH];
        float4 pp[BATCH];
#pragma unroll
        for (int j = 0; j < BATCH; ++j) {
          const int t = t0 + j * NT;
          oo[j] = -1;
          if (t < T) {
            const int o = (!use_bss && t < T2O_CAP) ? (int)C.t2o[t] : find_range(t);
            oo[j] = o;
            cc[j] = C.r_lo[o] + (t - C.r_off[o]);
            pp[j] = staged ? raw[t] : spos[cc[j]];
          }
        }
#pragma unroll
        for (int j = 0; j < BATCH; ++j) {
          if (oo[j] < 0) continue;
          const int o = oo[j], c = cc[j];
          const float4 p = pp[j];
          const int dest = C.adj[__float_as_int(p.w)][o] + (c - C.r_lo[o]) - F0;
          if (dest >= 0 && dest < CAND_CAP) {
            const float4 sh = C.r_shift[o];
            C.cand[dest] = make_float4(p.x + sh.x, p.y + sh.y, p.z + sh.z,
                                       __int_as_float(c | (C.r_code[o] << ANI_IMG_SHIFT)));
          }
        }
      }
      __syncthreads();
      tr.mark(TR_PLACE);
      // (d) the warps of this bucket compact their neighbours out of the window
      if (mine) {
        if (F0 == 0) {
          if (lane == 0) {
            s.seg_all[0] = 0;
            s.seg[0] = 0;
          }
          __syncwarp();
        }
        for (int sp = 0; sp < S; ++sp) {
          const int a = max(F0, C.off[sp * NRANGE]);
          const int b = min(F0 + CAND_CAP, C.off[(sp + 1) * NRANGE]);
          for (int base = a; base < b; base += 32) {
            const int idx = base + lane;
            const bool valid = idx < b;
            const float4 p = C.cand[valid ? idx - F0 : 0];
            const int word = __float_as_int(p.w);
            const float dx = p.x - pi.x, dy = p.y - pi.y, dz = p.z - pi.z;
            const float r2 = norm2(dx, dy, dz);
            const bool keep = valid && r2 <= rcr2 && word != (i | (13 << ANI_IMG_SHIFT));
            const unsigned m = __ballot_sync(ANI_FULL_MASK, keep);
            const int pos = cnt + __popc(m & lt);
            const bool stored = keep && pos < cap;
            // (an angular neighbour beyond the stored radial rows could not be addressed: the radial
            // overflow is reported instead)
            const bool keep_a = stored && r2 <= rca2;
            const unsigned ma = __ballot_sync(ANI_FULL_MASK, keep_a);
            if (stored) {
              s.nd[pos] = make_float4(dx, dy, dz, r2);  // the square root is taken once per neighbour below
              s.nj[pos] = word;
              if (keep_a) {
                const int pa = cnt_a + __popc(ma & lt);
                if (pa < ANI_MAX_ANG) s.aidx[pa] = (unsigned char)pos;
              }
            }
            cnt += __popc(m);
            cnt_a += __popc(ma);
          }
          // segment ends: partial while the species continues in the next window (rewritten then);
          // a species that ended before this window keeps the value it got there
          if (lane == 0 && C.off[(sp + 1) * NRANGE] >= F0) {
            s.seg_all[sp + 1] = min(cnt, cap);
            s.seg[sp + 1] = min(cnt_a, ANI_MAX_ANG);
          }
        }
      }
      __syncthreads();  // before the next window / phase overwrites the staging area
      tr.mark(TR_COMPACT);
    }
  }
  if (!has) return;
  atom_features<NA, NZ>(P, s, i, cnt, cnt_a, species_mask, row_of, aev, ldx, layout, nbr_cnt, nbr_list, cap, status,
                        tr);
  tr.write((size_t)(i - lo), lane);
}

// ---------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------
// The per-atom pieces of the backward pass.  k_aev_backward (one dE/dAEV row) and k_aev_backward_members (one row per
// ensemble member) are both sequences of these, so one member's arithmetic is that of the single-row kernel.
//
// The upstream gradient row lives in shared memory as the table {g_rad [RL], g_ang [pair_cap][GSTRIDE]}: g_ang is
// COMPACT, row = pair index among the elements present in the system (c1 <= c2 ranks), `pair_cap` rows; pairs beyond
// it (more elements than the launch was sized for) are read from the row in global memory.
constexpr int GSTRIDE = 36;  // floats per species-pair row: 16-byte aligned, rows 4 banks apart

template <class T>
__device__ __forceinline__ T* grad_table_ang(T* table, int RL) { return table + ((RL + 3) & ~3); }

__device__ __forceinline__ int compact_pair_row(int c1, int c2, int n_present) {
  return c1 * (2 * n_present - c1 + 1) / 2 + (c2 - c1);
}

__device__ __forceinline__ void copy_async4(float* dst_smem, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(dst_smem)), "l"(src)
               : "memory");
}

// Issue the cp.async copies of the upstream row `grow` into `table`; the caller commits the group.  Element pairs that
// do not occur in the system are never looked up (and never written by the MLP backward): walk the set bits of the
// element mask, (s1, s2 >= s1) pairs of present elements only.
__device__ __forceinline__ void stage_grad_row(const ani_aev_params& P, float* table, const float* grow,
                                               unsigned present, int n_present, int pair_cap) {
  const int lane = threadIdx.x & 31;
  const int S = P.num_species;
  const int RL = S * P.n_shf_r;
  float* g_ang = grad_table_ang(table, RL);
  for (int t = lane; t < RL; t += 32) copy_async4(table + t, grow + t);
  int c1 = 0;
  for (unsigned m1 = present; m1; m1 &= m1 - 1, ++c1) {
    const int s1 = __ffs(m1) - 1;
    const int base = s1 * (2 * S - s1 + 1) / 2 - s1;  // pair_index(s1, s2) = base + s2
    int c2 = c1;
    for (unsigned m2 = m1; m2; m2 &= m2 - 1, ++c2) {
      const int pp = base + __ffs(m2) - 1;
      const int cp = compact_pair_row(c1, c2, n_present);
      if (cp < pair_cap) copy_async4(g_ang + cp * GSTRIDE + lane, grow + RL + P.ang_pad + pp * 32 + lane);
    }
  }
}

// Geometry of atom i's neighbours, from the stored neighbour words or from the explicit rows `ex`: nd, nj, nsp, nfc,
// and the radial cutoff's derivative (once per neighbour, not once per (neighbour, shift) lane) into dfc[n * dfc_stride].
template <bool LAT>
__device__ __forceinline__ void backward_geometry(const ani_aev_params& P, const ani_grid& g, const WarpSmem& s,
                                                  const float4* __restrict__ spos, float4 pi, int i, int cnt,
                                                  const ExplicitNbrs& ex, int e0, const int32_t* __restrict__ nbr_list,
                                                  int cap, const float* __restrict__ lattice, int conf_i,
                                                  float* dfc_out, int dfc_stride) {
  const int lane = threadIdx.x & 31;
  for (int n = lane; n < cnt; n += 32) {
    int j;
    float4 dR;
    if (ex.start) {
      j = ex.j[e0 + n];
      dR = ex.d[e0 + n];
    } else {
      const int word = nbr_list[(size_t)i * cap + n];
      j = word & ANI_IDX_MASK;
      const int code = (unsigned)word >> ANI_IMG_SHIFT;
      const float4 p = spos[j];
      float3 sh = make_float3(0.f, 0.f, 0.f);
      if (code != 13) sh = LAT ? image_shift(lattice, conf_i, code) : image_shift(g, code);
      const float dx = (p.x + sh.x) - pi.x, dy = (p.y + sh.y) - pi.y, dz = (p.z + sh.z) - pi.z;
      dR = make_float4(dx, dy, dz, sqrtf(dx * dx + dy * dy + dz * dz));
    }
    s.nd[n] = dR;
    s.nj[n] = j;
    s.nsp[n] = (unsigned char)__float_as_int(spos[j].w);
    float fc, dfc;
    cutoff_value_grad(dR.w, P.rcr, P.cutoff_kind, fc, dfc);
    s.nfc[n] = fc;
    dfc_out[n * dfc_stride] = dfc;
  }
}

// Radial: dE/dR_n = sum_m g[s_n, m] * (G' fc + G fc'), then along the unit vector, into fgrad[3n .. 3n+2].  Lane =
// neighbour, serial over the shifts: no cross-lane reduction at all.
__device__ __forceinline__ void radial_backward(const ani_aev_params& P, const WarpSmem& s, int cnt,
                                                const float* table, const float* dfc_in, int dfc_stride) {
  const int lane = threadIdx.x & 31;
  const int nR = P.n_shf_r;
  for (int n = lane; n < cnt; n += 32) {
    const float4 d = s.nd[n];
    const float fc = s.nfc[n], dfc = dfc_in[n * dfc_stride];
    const float* __restrict__ gr = table + s.nsp[n] * nR;
    float acc = 0.f;
#pragma unroll 4
    for (int m = 0; m < nR; ++m) {
      const float x = d.w - P.shf_r[m];
      const float G = 0.25f * fast_exp(-P.eta_r * x * x);
      acc = fmaf(gr[m] * G, fmaf(-2.0f * P.eta_r * x, fc, dfc), acc);
    }
    const float sc = d.w > 1e-10f ? acc * fast_rcp(d.w) : 0.f;
    s.fgrad[3 * n + 0] = sc * d.x;
    s.fgrad[3 * n + 1] = sc * d.y;
    s.fgrad[3 * n + 2] = sc * d.z;
  }
}

// Angular: adds dE/dr_j of the n_ang neighbours of the angular list to fgrad.  Lanes own rows j of the list.
// CONSTS_IN_REGS: the angular constants (shf_a, cos_z, sin_z) are copied into registers; otherwise they are read from
// the kernel parameters as constant-bank operands, which keeps the member loop of k_aev_backward_members within its
// register budget.  SHAPE_IN_REGS: likewise for the element count and the radial width that
// address pairs beyond the table.  Both are register-allocation choices of the calling kernel; they change no result.
template <int NA, int NZ, bool CONSTS_IN_REGS, bool SHAPE_IN_REGS>
__device__ __forceinline__ void angular_backward(const ani_aev_params& P, const WarpSmem& s, int n_ang,
                                                 const float* table, const float* grow, unsigned present, int n_present,
                                                 int pair_cap) {
  const int lane = threadIdx.x & 31;
  if (n_ang < 2) return;
  const int S_reg = P.num_species;
  const int RL_reg = S_reg * P.n_shf_r;
  const float* g_ang = grad_table_ang(table, RL_reg);
  float shfA[NA], cz[NZ], sz[NZ];
  if (CONSTS_IN_REGS) {
#pragma unroll
    for (int a = 0; a < NA; ++a) shfA[a] = P.shf_a[a];
#pragma unroll
    for (int z = 0; z < NZ; ++z) {
      cz[z] = P.cos_z[z];
      sz[z] = P.sin_z[z];
    }
  }
  // The three sums every pair needs (symmetric in j <-> k):
  //   S0 = sum g f1 f2,  S1 = sum g f1' f2 (d/dcos),  S2 = sum g f1 f2' (d/dRbar)
  auto pair_sums = [&](const float4& dj, const float4& dk, int sj, int sk, float& cosT, float& inv_rr, float& S0,
                       float& S1, float& S2) {
    const float dot = dj.x * dk.x + dj.y * dk.y + dj.z * dk.z;
    inv_rr = fast_rcp(fmaxf(dj.w * dk.w, 1e-10f));
    cosT = dot * inv_rr;
    const float c = 0.95f * cosT;
    const float sn = fast_sqrt(fmaxf(1.0f - c * c, 0.f));
    const float c_over_s = c * fast_rcp(sn);
    const float rbar = 0.5f * (dj.w + dk.w);
    // t_z = sum_a g[a,z] f2[a],  u_z = sum_a g[a,z] f2'[a]: the 32 upstream values of this pair are
    // one 16-byte-aligned row -> 8 vector loads, from the compact table or, beyond it, from the row in global memory
    const int cj = __popc(present & ((1u << sj) - 1u)), ck = __popc(present & ((1u << sk) - 1u));
    const int cp = compact_pair_row(min(cj, ck), max(cj, ck), n_present);
    const float4* __restrict__ gp =
        cp < pair_cap ? reinterpret_cast<const float4*>(g_ang + cp * GSTRIDE)
                      : reinterpret_cast<const float4*>(grow + (SHAPE_IN_REGS ? RL_reg : P.num_species * P.n_shf_r) + P.ang_pad +
                                                         pair_index(sj, sk, SHAPE_IN_REGS ? S_reg : P.num_species) * 32);
    float tz[NZ], uz[NZ];
#pragma unroll
    for (int z = 0; z < NZ; ++z) tz[z] = uz[z] = 0.f;
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      const float d = rbar - (CONSTS_IN_REGS ? shfA[a] : P.shf_a[a]);
      const float f2 = fast_exp(-P.eta_a * d * d);
      const float f2p = -2.0f * P.eta_a * d * f2;
#pragma unroll
      for (int q = 0; q < NZ / 4; ++q) {
        const float4 gv = gp[a * (NZ / 4) + q];
        tz[4 * q + 0] = fmaf(gv.x, f2, tz[4 * q + 0]);
        tz[4 * q + 1] = fmaf(gv.y, f2, tz[4 * q + 1]);
        tz[4 * q + 2] = fmaf(gv.z, f2, tz[4 * q + 2]);
        tz[4 * q + 3] = fmaf(gv.w, f2, tz[4 * q + 3]);
        uz[4 * q + 0] = fmaf(gv.x, f2p, uz[4 * q + 0]);
        uz[4 * q + 1] = fmaf(gv.y, f2p, uz[4 * q + 1]);
        uz[4 * q + 2] = fmaf(gv.z, f2p, uz[4 * q + 2]);
        uz[4 * q + 3] = fmaf(gv.w, f2p, uz[4 * q + 3]);
      }
    }
    S0 = S1 = S2 = 0.f;
#pragma unroll
    for (int z = 0; z < NZ; ++z) {
      const float cosz = CONSTS_IN_REGS ? cz[z] : P.cos_z[z], sinz = CONSTS_IN_REGS ? sz[z] : P.sin_z[z];
      const float base = fmaxf(0.5f * (1.0f + c * cosz + sn * sinz), 0.f);
      const float lg = fast_log2(base);
      const float f1 = fast_exp2(P.zeta * lg);
      const float pw1 = fast_exp2((P.zeta - 1.0f) * lg);
      const float f1p = P.zeta * pw1 * (0.475f * (cosz - c_over_s * sinz));
      S0 = fmaf(f1, tz[z], S0);
      S1 = fmaf(f1p, tz[z], S1);
      S2 = fmaf(f1, uz[z], S2);
    }
  };
  int lpr = 1;
  while (lpr * 2 * n_ang <= 32) lpr *= 2;
  const int sub = lane % lpr;
  if (n_ang <= 32) {
    // Rotation over UNORDERED pairs: in step t row j evaluates the pair (j, (j + t) mod n) once,
    // keeps its own share and hands the partner's share to the lane that owns row k with one
    // shuffle (every row receives from row j - t at the same step).  t runs to n/2; for even n
    // the last step would see every pair from both ends, so only rows j < n/2 take part in it.
    // The lpr lanes of a row split the steps.  Half the transcendental work of ordered pairs.
    const int j = lane / lpr;
    const bool jvalid = j < n_ang;
    const int half_n = n_ang >> 1;
    const bool even = (n_ang & 1) == 0;
    float gx = 0.f, gy = 0.f, gz = 0.f;
    int nj_ = 0, sj = 0;
    float4 dj = make_float4(0.f, 0.f, 0.f, 1.f);
    float fcj = 0.f, dfcj = 0.f, inv_rj = 0.f;
    if (jvalid) {
      nj_ = s.aidx[j];
      dj = s.nd[nj_];
      fcj = s.afc[j];
      dfcj = s.afcd[j];
      sj = s.nsp[nj_];
      inv_rj = dj.w > 1e-10f ? fast_rcp(dj.w) : 0.f;
    }
    const int steps = (half_n + lpr - 1) / lpr;
    for (int it = 0; it < steps; ++it) {
      const int t = 1 + it * lpr + sub;
      const bool active = jvalid && t <= half_n && !(even && t == half_n && j >= half_n);
      float px = 0.f, py = 0.f, pz = 0.f;
      if (active) {
        int k = j + t;
        if (k >= n_ang) k -= n_ang;
        const int nk_ = s.aidx[k];
        const float4 dk = s.nd[nk_];
        const float fck = s.afc[k], dfck = s.afcd[k];
        const float inv_rk = dk.w > 1e-10f ? fast_rcp(dk.w) : 0.f;
        float cosT, inv_rr, S0, S1, S2;
        pair_sums(dj, dk, sj, (int)s.nsp[nk_], cosT, inv_rr, S0, S1, S2);
        // feature = 2 f1 f2 fcj fck (once per unordered pair): its derivative with respect to
        // r_j is this lane's share, the one with respect to r_k goes to the partner row
        const float W = fcj * fck;
        const float dEdcos = 2.0f * W * S1;
        const float dEdRj = S2 * W + 2.0f * S0 * dfcj * fck;
        const float dEdRk = S2 * W + 2.0f * S0 * fcj * dfck;
        const float coefj = (dEdRj - dEdcos * cosT * inv_rj) * inv_rj;
        const float coefk = (dEdRk - dEdcos * cosT * inv_rk) * inv_rk;
        const float coefx = dEdcos * inv_rr;
        gx += coefj * dj.x + coefx * dk.x;
        gy += coefj * dj.y + coefx * dk.y;
        gz += coefj * dj.z + coefx * dk.z;
        px = coefk * dk.x + coefx * dj.x;
        py = coefk * dk.y + coefx * dj.y;
        pz = coefk * dk.z + coefx * dj.z;
      }
      int src_row = j - t;
      if (src_row < 0) src_row += n_ang;
      const int src_lane = jvalid ? src_row * lpr + sub : lane;
      const float rx = __shfl_sync(ANI_FULL_MASK, px, src_lane);
      const float ry = __shfl_sync(ANI_FULL_MASK, py, src_lane);
      const float rz = __shfl_sync(ANI_FULL_MASK, pz, src_lane);
      if (jvalid) {  // inactive sources sent zeros
        gx += rx;
        gy += ry;
        gz += rz;
      }
    }
    for (int o = lpr / 2; o > 0; o >>= 1) {
      gx += __shfl_xor_sync(ANI_FULL_MASK, gx, o);
      gy += __shfl_xor_sync(ANI_FULL_MASK, gy, o);
      gz += __shfl_xor_sync(ANI_FULL_MASK, gz, o);
    }
    if (jvalid && sub == 0) {
      s.fgrad[3 * nj_ + 0] += gx;
      s.fgrad[3 * nj_ + 1] += gy;
      s.fgrad[3 * nj_ + 2] += gz;
    }
  } else {
    // more rows than lanes: ordered pairs (j, k), several passes of 32 rows
    for (int row0 = 0; row0 < n_ang; row0 += 32) {
      const int j = row0 + lane;
      float gx = 0.f, gy = 0.f, gz = 0.f;
      if (j < n_ang) {
        const int nj_ = s.aidx[j];
        const float4 dj = s.nd[nj_];
        const float fcj = s.afc[j], dfcj = s.afcd[j];
        const int sj = s.nsp[nj_];
        const float inv_rj = dj.w > 1e-10f ? fast_rcp(dj.w) : 0.f;
        for (int k = 0; k < n_ang; ++k) {
          if (k == j) continue;
          const int nk_ = s.aidx[k];
          const float4 dk = s.nd[nk_];
          const float fck = s.afc[k];
          float cosT, inv_rr, S0, S1, S2;
          pair_sums(dj, dk, sj, (int)s.nsp[nk_], cosT, inv_rr, S0, S1, S2);
          const float W = fcj * fck;
          const float dEdRj = S2 * W + 2.0f * S0 * dfcj * fck;  // 2*(0.5*S2*W + S0*fcj'*fck)
          const float dEdcos = 2.0f * W * S1;
          const float coefj = (dEdRj - dEdcos * cosT * inv_rj) * inv_rj;
          const float coefk = dEdcos * inv_rr;
          gx += coefj * dj.x + coefk * dk.x;
          gy += coefj * dj.y + coefk * dk.y;
          gz += coefj * dj.z + coefk * dk.z;
        }
        s.fgrad[3 * nj_ + 0] += gx;
        s.fgrad[3 * nj_ + 1] += gy;
        s.fgrad[3 * nj_ + 2] += gz;
      }
    }
  }
}

// Scatter into `grad`: neighbour j gets +dE_i/dr_j, the centre atom i minus the sum.
// VIRIAL: W_ab += (dE_i/dDelta_in)_a (Delta_in)_b, the "f dot r" virial of ase.py:164-168 (dE/dDelta^T @ Delta over
// the pairs); ANI_VIRIAL_SLOTS partial sums keep the atomics apart.
template <bool VIRIAL, bool LAT>
__device__ __forceinline__ void scatter_backward(const ani_grid& g, const WarpSmem& s, int cnt,
                                                 const int32_t* __restrict__ sorted_orig, int i, int conf_i,
                                                 float* __restrict__ grad, double* __restrict__ virial) {
  const int lane = threadIdx.x & 31;
  float sx = 0.f, sy = 0.f, sz_ = 0.f;
  float vir[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) vir[k] = 0.f;
  for (int n = lane; n < cnt; n += 32) {
    const float fx = s.fgrad[3 * n], fy = s.fgrad[3 * n + 1], fz = s.fgrad[3 * n + 2];
    const int oj = sorted_orig[s.nj[n]];
    atomicAdd(&grad[3 * (size_t)oj + 0], fx);
    atomicAdd(&grad[3 * (size_t)oj + 1], fy);
    atomicAdd(&grad[3 * (size_t)oj + 2], fz);
    sx += fx;
    sy += fy;
    sz_ += fz;
    if (VIRIAL) {
      const float4 d = s.nd[n];
      vir[0] = fmaf(fx, d.x, vir[0]); vir[1] = fmaf(fx, d.y, vir[1]); vir[2] = fmaf(fx, d.z, vir[2]);
      vir[3] = fmaf(fy, d.x, vir[3]); vir[4] = fmaf(fy, d.y, vir[4]); vir[5] = fmaf(fy, d.z, vir[5]);
      vir[6] = fmaf(fz, d.x, vir[6]); vir[7] = fmaf(fz, d.y, vir[7]); vir[8] = fmaf(fz, d.z, vir[8]);
    }
  }
  if (VIRIAL && virial) {
    // a periodic batch (modes 2, 3) keeps one set of slots per conformer: the conformer of the central atom
    const int conf = LAT ? conf_i : g.mode == 2 ? sorted_orig[i] / g.n_per_conf : 0;
    double* slots = virial + (size_t)conf * ANI_VIRIAL_SLOTS * 9;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const float v = warp_sum(vir[k]);
      if (lane == 0) atomicAdd(&slots[(blockIdx.x % ANI_VIRIAL_SLOTS) * 9 + k], (double)v);
    }
  }
  sx = warp_sum(sx);
  sy = warp_sum(sy);
  sz_ = warp_sum(sz_);
  if (lane == 0) {
    const int oi = sorted_orig[i];
    atomicAdd(&grad[3 * (size_t)oi + 0], -sx);
    atomicAdd(&grad[3 * (size_t)oi + 1], -sy);
    atomicAdd(&grad[3 * (size_t)oi + 2], -sz_);
  }
}

// Backward (forces) of one dE/dAEV row per atom: the row's cp.async copies are in flight while the neighbour geometry
// is rebuilt; radial; angular list; angular; scatter.  LAT (grid mode 3): image shifts in the lattice of the central
// atom's conformer (lattice table)
template <int NA, int NZ, bool VIRIAL = false, bool LAT = false>
__global__ void __launch_bounds__(AEV_WARPS * 32, ANI_AEV_BWD_MIN_CTAS)
    k_aev_backward(const __grid_constant__ ani_aev_params P, const ani_grid* __restrict__ grid,
                   const float4* __restrict__ spos, const int32_t* __restrict__ sorted_orig, int lo, int hi,
                   const int32_t* __restrict__ row_of, const float* __restrict__ gaev, int ldx,
                   const int32_t* __restrict__ nbr_cnt, const int32_t* __restrict__ nbr_list, const ExplicitNbrs ex,
                   const int32_t* __restrict__ species_mask, int cap, float* __restrict__ grad_coords,
                   int32_t* __restrict__ status, size_t warp_bytes, int pair_cap, double* __restrict__ virial,
                   const float* __restrict__ lattice) {
  static_assert(NA * NZ == 32, "one lane per angular feature");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const ani_grid g = *grid;
  hi = min(hi, g.n_real);
  const int i = lo + blockIdx.x * AEV_WARPS + warp;
  if (i >= hi) return;
  const WarpSmem s = carve(smem_raw + warp * warp_bytes, cap, true);
  const unsigned present = (species_mask ? (unsigned)species_mask[0] : 0xffffffffu) & ((1u << P.num_species) - 1u);
  const int n_present = __popc(present);
  const float* grow = gaev + (size_t)row_of[i] * ldx;
  stage_grad_row(P, s.rad, grow, present, n_present, pair_cap);
  asm volatile("cp.async.commit_group;" ::: "memory");

  const float4 pi = spos[i];
  if (__float_as_int(pi.w) < 0) return;  // padding atom (explicit neighbour rows only)
  const int e0 = ex.start ? ex.start[i] : 0;
  const int cnt = ex.start ? min(ex.start[i + 1] - e0, cap) : nbr_cnt[i];
  const int conf_i = LAT ? sorted_orig[i] / g.n_per_conf : 0;   // neighbours lie in the centre's conformer
  // dfc is parked in fgrad[3n] until the radial pass overwrites fgrad[3n .. 3n+2]
  backward_geometry<LAT>(P, g, s, spos, pi, i, cnt, ex, e0, nbr_list, cap, lattice, conf_i, s.fgrad, 3);
  asm volatile("cp.async.wait_all;" ::: "memory");  // the upstream gradient row has landed
  __syncwarp();
  radial_backward(P, s, cnt, s.rad, s.fgrad, 3);
  __syncwarp();
  const int n_ang = compact_angular_list(P, s, cnt, lane, status);
  angular_backward<NA, NZ, true, VIRIAL>(P, s, n_ang, s.rad, grow, present, n_present, pair_cap);
  __syncwarp();
  scatter_backward<VIRIAL, LAT>(g, s, cnt, sorted_orig, i, conf_i, grad_coords, virial);
}

// ---------------------------------------------------------------------------------------
// backward of every ensemble member in one launch (query-by-committee statistics)
// ---------------------------------------------------------------------------------------
// Active members of an ani_b200_aev_backward_members call: output k contracts slab idx[k]
struct MemberSlabs : ActiveMembers {
  long long stride;  // floats between the dE/dAEV slabs of consecutive members
};

// The pieces of k_aev_backward with the per-member ones in a loop.  A warp rebuilds its atom's neighbour geometry
// (backward_geometry, compact_angular_list) once; then, for k = 0 .. count - 1, it contracts member idx[k]'s dE/dAEV
// row (radial_backward, angular_backward) and scatters into grad_members[k] (scatter_backward).  The rows are staged in two
// shared-memory tables with stage_grad_row: member k + 1's row is in flight while member k is contracted, so shared
// memory per warp does not depend on the number of members; dfc has its own array after them (fgrad is rewritten per
// member).  The arithmetic of one member is that of k_aev_backward (same order within an atom): only the order of the
// float atomics differs.  No explicit neighbour rows and no virial.
template <int NA, int NZ, bool LAT = false>
__global__ void __launch_bounds__(AEV_WARPS * 32, NA == 8 ? ANI_AEV_BWD_MEMBERS_MIN_CTAS : ANI_AEV_BWD_MEMBERS_MIN_CTAS - 1)
    k_aev_backward_members(const __grid_constant__ ani_aev_params P, const ani_grid* __restrict__ grid,
                           const float4* __restrict__ spos, const int32_t* __restrict__ sorted_orig, int lo, int hi,
                           const int32_t* __restrict__ row_of, const float* __restrict__ slabs, int ldx,
                           const int32_t* __restrict__ nbr_cnt, const int32_t* __restrict__ nbr_list,
                           const int32_t* __restrict__ species_mask, int cap, float* __restrict__ grad_members,
                           long long grad_stride, int32_t* __restrict__ status, size_t warp_bytes, int pair_cap,
                           int gbuf_floats, const float* __restrict__ lattice, const __grid_constant__ MemberSlabs ms) {
  static_assert(NA * NZ == 32, "one lane per angular feature");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const ani_grid g = *grid;
  hi = min(hi, g.n_real);
  const int i = lo + blockIdx.x * AEV_WARPS + warp;
  if (i >= hi) return;
  const WarpSmem s = carve(smem_raw + warp * warp_bytes, cap, true);
  const unsigned present = (species_mask ? (unsigned)species_mask[0] : 0xffffffffu) & ((1u << P.num_species) - 1u);
  const int n_present = __popc(present);
  // [table 0 | table 1] of gbuf_floats each, then dfc(R; Rcr) per neighbour
  float* ndfc = s.rad + 2 * gbuf_floats;
  const size_t row = (size_t)row_of[i] * ldx;
  auto member_row = [&](int k) { return slabs + (size_t)ms.idx[k] * ms.stride + row; };
  // member k's row -> table k & 1 (one commit group per member; an empty group past the last member)
  auto stage = [&](int k) {
    if (k < ms.count) stage_grad_row(P, s.rad + (k & 1) * gbuf_floats, member_row(k), present, n_present, pair_cap);
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  stage(0);

  const int cnt = nbr_cnt[i];
  const int conf_i = LAT ? sorted_orig[i] / g.n_per_conf : 0;
  backward_geometry<LAT>(P, g, s, spos, spos[i], i, cnt, ExplicitNbrs{nullptr, nullptr, nullptr}, 0, nbr_list, cap,
                         lattice, conf_i, ndfc, 1);
  __syncwarp();
  const int n_ang = compact_angular_list(P, s, cnt, lane, status);

  for (int k = 0; k < ms.count; ++k) {
    stage(k + 1);
    asm volatile("cp.async.wait_group 1;" ::: "memory");  // member k's row has landed
    __syncwarp();
    const float* table = s.rad + (k & 1) * gbuf_floats;
    radial_backward(P, s, cnt, table, ndfc, 1);
    __syncwarp();
    angular_backward<NA, NZ, false, true>(P, s, n_ang, table, member_row(k), present, n_present, pair_cap);
    __syncwarp();
    scatter_backward<false, LAT>(g, s, cnt, sorted_orig, i, conf_i, grad_members + (size_t)k * grad_stride,
                                 nullptr);
    __syncwarp();  // fgrad and table k & 1 are rewritten by the next member
  }
}

// ---------------------------------------------------------------------------------------
// reference-format half neighbour list (API parity path; one thread per atom)
// ---------------------------------------------------------------------------------------
template <bool FILL>
__global__ void k_half_list(const ani_grid* __restrict__ grid, const int32_t* __restrict__ bin_start,
                            const float4* __restrict__ spos, const int32_t* __restrict__ sbin,
                            const int32_t* __restrict__ sorted_orig, int n, float cutoff,
                            int32_t* __restrict__ pair_count, const int32_t* __restrict__ pair_start,
                            long long cap, int64_t* __restrict__ idx0, int64_t* __restrict__ idx1,
                            float* __restrict__ distances, float* __restrict__ diffs,
                            int32_t* __restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const ani_grid g = *grid;
  int count = 0;
  if (i < g.n_real) {
    const float4 pi = spos[i];
    const int oi = sorted_orig[i];
    const float c2 = cutoff * cutoff;
    long long out = FILL ? (long long)pair_start[i] : 0;
    const int b = sbin[i];
    int ix = 0, iy = 0, iz = 0, span = 0, base = 0;
    if (g.mode != 1) {
      base = bucket_coords(g, b, ix, iy, iz);
      span = 1;
    }
    for (int ox = -span; ox <= span; ++ox)
      for (int oy = -span; oy <= span; ++oy)
        for (int oz = -span; oz <= span; ++oz) {
          NeighbourRange r;
          if (g.mode != 1) {
            if (!neighbour_bucket(g, bin_start, base, ix, iy, iz, ox, oy, oz, r)) continue;
          } else {
            r.lo = bin_start[b];
            r.hi = bin_start[b + 1];
            r.code = 13;
          }
          const float3 sh = (r.code == 13) ? make_float3(0.f, 0.f, 0.f) : image_shift(g, r.code);
          for (int c = r.lo; c < r.hi; ++c) {
            const int oj = sorted_orig[c];
            // every unordered pair is seen from both ends; keep it at the lower input index
            // (self-image pairs: keep the upper half of the image codes)
            if (!(oi < oj || (oi == oj && r.code > 13))) continue;
            const float4 p = spos[c];
            const float dx = pi.x - (p.x + sh.x), dy = pi.y - (p.y + sh.y), dz = pi.z - (p.z + sh.z);
            const float r2 = dx * dx + dy * dy + dz * dz;
            if (r2 > c2) continue;
            if (FILL) {
              if (out < cap) {
                idx0[out] = oi;
                idx1[out] = oj;
                distances[out] = sqrtf(r2);
                diffs[3 * out + 0] = dx;
                diffs[3 * out + 1] = dy;
                diffs[3 * out + 2] = dz;
              } else {
                atomicOr(status, ANI_STATUS_PAIR_OVERFLOW);
              }
              ++out;
            }
            ++count;
          }
        }
  }
  if (!FILL) pair_count[i] = count;
}

// exclusive scan of an int array by one block: out[0..m], out[m] = total
__global__ void k_scan_i32(const int32_t* __restrict__ in, int m, int32_t* __restrict__ out) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < m; base += blockDim.x) {
    const int i = base + tid;
    const int v = (i < m) ? in[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(ANI_FULL_MASK, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[w] = x;
    __syncthreads();
    if (w == 0) {
      int t = (lane < (blockDim.x >> 5)) ? s_warp[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(ANI_FULL_MASK, t, o);
        if (lane >= o) t += y;
      }
      s_warp[lane] = t;
    }
    __syncthreads();
    const int incl = x + ((w == 0) ? 0 : s_warp[w - 1]) + s_carry;
    if (i < m) out[i] = incl - v;
    __syncthreads();
    if (tid == blockDim.x - 1) s_carry = incl;
    __syncthreads();
  }
  if (tid == 0) out[m] = s_carry;
}

static int check_params(const ani_aev_params* p) {
  if (!p) return ANI_ERR_BAD_ARG;
  if (p->num_species < 1 || p->num_species > ANI_MAX_SPECIES) return ANI_ERR_UNSUPPORTED;
  if (p->n_shf_r < 1 || p->n_shf_r > ANI_MAX_SHFR) return ANI_ERR_UNSUPPORTED;
  if (!((p->n_shf_a == 8 && p->n_shf_z == 4) || (p->n_shf_a == 4 && p->n_shf_z == 8)))
    return ANI_ERR_UNSUPPORTED;  // one lane per angular feature: ShfA x ShfZ must be 8x4 or 4x8
  if (!(p->rca < p->rcr) || p->rca <= 0.f) return ANI_ERR_BAD_ARG;  // aev/_computer.py:233
  if (!(p->zeta > 1.0f)) return ANI_ERR_UNSUPPORTED;
  if (p->cutoff_kind != 0 && p->cutoff_kind != 1) return ANI_ERR_UNSUPPORTED;
  return ANI_OK;
}

// the template instance of an AEV kernel for the angular shape (ShfA x ShfZ) and grid mode 3 (lattice table)
template <int NA_, bool LAT_>
struct AevShape {
  static constexpr int NA = NA_, NZ = 32 / NA_;
  static constexpr bool LAT = LAT_;
};
template <class F>
static void dispatch_shape(const ani_aev_params* params, bool lattice, F&& f) {
  if (params->n_shf_a == 8)
    lattice ? f(AevShape<8, true>{}) : f(AevShape<8, false>{});
  else
    lattice ? f(AevShape<4, true>{}) : f(AevShape<4, false>{});
}

// ---- launchers shared by the bucket-grid and the explicit-pair-list entry points -----------
static int launch_aev_forward(const ani_aev_params* params, const ani_grid* grid, const int32_t* bin_start,
                              const float* spos, const int32_t* sbin, const float* bucket_ranges,
                              const int32_t* bucket_species, const int32_t* species_mask, ExplicitNbrs ex, int n, int lo, int hi,
                              const int32_t* row_of, float* aev, int ldx, int layout, int32_t* nbr_cnt,
                              int32_t* nbr_list, int nbr_cap, int32_t* status, void* stream,
                              const float* lattice = nullptr) {
  int rc = check_params(params);
  if (rc != ANI_OK) return rc;
  if (!grid || !spos || !row_of || !aev || !status) return ANI_ERR_BAD_ARG;
  if (lo < 0 || hi > n || lo > hi) return ANI_ERR_BAD_ARG;
  if (nbr_cap < 32 || nbr_cap > 256 || nbr_cap % 32) return ANI_ERR_BAD_ARG;
  const int out_dim = params->num_species * params->n_shf_r +
                      params->num_species * (params->num_species + 1) / 2 * 32;
  if (ldx < out_dim) return ANI_ERR_BAD_ARG;
  if (layout != 0 && layout != 1) return ANI_ERR_BAD_ARG;
  if (layout == 1 && ldx % 32) return ANI_ERR_BAD_ARG;
  if (hi == lo) return ANI_OK;
  const size_t wb = warp_smem_bytes(nbr_cap, 0, false);
  cudaStream_t st = (cudaStream_t)stream;
  const float4* sp4 = reinterpret_cast<const float4*>(spos);
  const float4* rng4 = reinterpret_cast<const float4*>(bucket_ranges);
  // bucket-grid path: CTA-staged neighbourhoods (ANI_B200_AEV_LEGACY=1 keeps the warp-per-atom search
  // of k_aev_forward, which also serves the explicit neighbour rows)
  static const bool legacy = []() {
    const char* e = getenv("ANI_B200_AEV_LEGACY");
    return e && atoi(e) != 0;
  }();
  // ANI_B200_AEV_TMA=1: stage the candidate ranges of a CTA's first bucket with TMA bulk copies (cp.async.bulk +
  // mbarrier) instead of per-thread global loads.  Same results; off by default: 27 copies of ~220 bytes per CTA are
  // small for the copy engine and every thread of the CTA idles on the mbarrier, where the batched per-thread loads
  // overlap with their own bookkeeping.
  static const int tma_stage = []() {
    const char* e = getenv("ANI_B200_AEV_TMA");
    return e && atoi(e) != 0 ? 1 : 0;
  }();
  const bool staged = !ex.start && !legacy;
  const int warps = staged ? AEV_FWD_WARPS : AEV_WARPS;
  const size_t smem = wb * warps;
  const int blocks = (hi - lo + warps - 1) / warps;
  auto go = [&](auto k, auto... args) {
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k<<<blocks, warps * 32, smem, st>>>(args...);
  };
  dispatch_shape(params, lattice != nullptr, [&](auto sh) {
    using Sh = decltype(sh);
    if (staged) {
      auto k = tma_stage ? k_aev_forward_cta<Sh::NA, Sh::NZ, true, Sh::LAT> : k_aev_forward_cta<Sh::NA, Sh::NZ, false, Sh::LAT>;
      go(k, *params, grid, bin_start, sp4, sbin, rng4, species_mask, lo, hi, row_of, aev, ldx, layout, nbr_cnt,
         nbr_list, nbr_cap, status, wb, tma_stage, bucket_species, lattice);
    } else {
      go(k_aev_forward<Sh::NA, Sh::NZ, Sh::LAT>, *params, grid, bin_start, sp4, sbin, rng4, species_mask, ex, lo, hi,
         row_of, aev, ldx, layout, nbr_cnt, nbr_list, nbr_cap, status, wb, lattice);
    }
  });
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

// ---- backward launchers -------------------------------------------------------------------
static int check_backward_args(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                               const int32_t* sorted_orig, int n, int lo, int hi, const int32_t* row_of,
                               const float* grad_aev, const float* grad_out, const int32_t* status, int nbr_cap) {
  int rc = check_params(params);
  if (rc != ANI_OK) return rc;
  if (!grid || !spos || !sorted_orig || !row_of || !grad_aev || !grad_out || !status) return ANI_ERR_BAD_ARG;
  if (lo < 0 || hi > n || lo > hi) return ANI_ERR_BAD_ARG;
  if (nbr_cap < 32 || nbr_cap > 256 || nbr_cap % 32) return ANI_ERR_BAD_ARG;
  return ANI_OK;
}

// The shared-memory gradient table {g_rad, g_ang [pair_cap][GSTRIDE]} of the backward kernels.  Its rows are every
// element pair, or the pairs of `max_elements` elements when the caller knows the composition (more elements at run
// time still work: those pairs are read from global memory).  pair_sums reads the pairs beyond the table as float4 runs
// of the upstream row, which needs the angular block 16-byte aligned in every row: RL + ang_pad, ldx and the stride
// between slabs multiples of 4 (not so for, e.g., 7 elements x 15 shifts without ang_pad).  Otherwise the table holds
// every pair and global memory is never read there.
struct GradTable {
  int pair_cap;
  int floats;
};
static GradTable grad_table(const ani_aev_params* params, const int32_t* species_mask, int max_elements,
                            const float* grad_aev, int ldx, long long slab_stride) {
  const int S = params->num_species;
  const int RL = S * params->n_shf_r;
  const int E = (max_elements > 0 && max_elements < S) ? max_elements : S;
  const bool ang_aligned = (RL + params->ang_pad) % 4 == 0 && ldx % 4 == 0 && ((uintptr_t)grad_aev & 15) == 0 &&
                           slab_stride % 4 == 0;
  const int pair_cap = (species_mask && ang_aligned) ? E * (E + 1) / 2 : S * (S + 1) / 2;
  return GradTable{pair_cap, ((RL + 3) & ~3) + GSTRIDE * pair_cap};
}

static int launch_aev_backward(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                               const int32_t* sorted_orig, int n, int lo, int hi, const int32_t* row_of,
                               const float* grad_aev, int ldx, const int32_t* nbr_cnt, const int32_t* nbr_list,
                               ExplicitNbrs ex, const int32_t* species_mask, int nbr_cap, float* grad_coords,
                               int32_t* status, void* stream, int max_elements = 0, double* virial = nullptr,
                               const float* lattice = nullptr) {
  int rc = check_backward_args(params, grid, spos, sorted_orig, n, lo, hi, row_of, grad_aev, grad_coords, status,
                               nbr_cap);
  if (rc != ANI_OK) return rc;
  if (hi == lo) return ANI_OK;
  const GradTable t = grad_table(params, species_mask, max_elements, grad_aev, ldx, ldx);
  const size_t wb = warp_smem_bytes(nbr_cap, t.floats, true);
  const size_t smem = wb * AEV_WARPS;
  const int blocks = (hi - lo + AEV_WARPS - 1) / AEV_WARPS;
  cudaStream_t st = (cudaStream_t)stream;
  const float4* sp4 = reinterpret_cast<const float4*>(spos);
  auto go = [&](auto k) {
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k<<<blocks, AEV_WARPS * 32, smem, st>>>(*params, grid, sp4, sorted_orig, lo, hi, row_of, grad_aev, ldx, nbr_cnt,
                                            nbr_list, ex, species_mask, nbr_cap, grad_coords, status, wb, t.pair_cap,
                                            virial, lattice);
  };
  dispatch_shape(params, lattice, [&](auto sh) {
    using Sh = decltype(sh);
    if (virial)
      go(k_aev_backward<Sh::NA, Sh::NZ, true, Sh::LAT>);
    else
      go(k_aev_backward<Sh::NA, Sh::NZ, false, Sh::LAT>);
  });
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

static int launch_aev_backward_members(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                                       const int32_t* sorted_orig, const int32_t* species_mask, int n, int lo, int hi,
                                       const int32_t* row_of, const float* slabs, int ldx, long long slab_stride,
                                       const int32_t* members, int n_members, const int32_t* nbr_cnt,
                                       const int32_t* nbr_list, int nbr_cap, float* grad_members, int32_t* status,
                                       int max_elements, const float* lattice, void* stream) {
  int rc = check_backward_args(params, grid, spos, sorted_orig, n, lo, hi, row_of, slabs, grad_members, status,
                               nbr_cap);
  if (rc != ANI_OK) return rc;
  if (!nbr_cnt || !nbr_list) return ANI_ERR_BAD_ARG;
  if (n_members < 1 || slab_stride < (long long)ldx) return ANI_ERR_BAD_ARG;
  MemberSlabs ms;
  rc = active_members(members, n_members, ms);
  if (rc != ANI_OK) return rc;
  ms.stride = slab_stride;
  if (hi == lo) return ANI_OK;
  // two gradient tables (double-buffered rows), plus dfc per neighbour
  const GradTable t = grad_table(params, species_mask, max_elements, slabs, ldx, slab_stride);
  const size_t wb = warp_smem_bytes(nbr_cap, 2 * t.floats + nbr_cap, true);
  const size_t smem = wb * AEV_WARPS;
  const int blocks = (hi - lo + AEV_WARPS - 1) / AEV_WARPS;
  cudaStream_t st = (cudaStream_t)stream;
  const float4* sp4 = reinterpret_cast<const float4*>(spos);
  dispatch_shape(params, lattice, [&](auto sh) {
    using Sh = decltype(sh);
    auto k = k_aev_backward_members<Sh::NA, Sh::NZ, Sh::LAT>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k<<<blocks, AEV_WARPS * 32, smem, st>>>(*params, grid, sp4, sorted_orig, lo, hi, row_of, slabs, ldx, nbr_cnt,
                                            nbr_list, species_mask, nbr_cap, grad_members, 3LL * n, status, wb,
                                            t.pair_cap, t.floats, lattice, ms);
  });
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

// ---- half pair list -> per-atom rows (both directions) ------------------------------------
__global__ void k_pairs_count(const int64_t* __restrict__ idx0, const int64_t* __restrict__ idx1, long long P,
                              int32_t* __restrict__ counts) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  atomicAdd(&counts[idx0[p]], 1);
  atomicAdd(&counts[idx1[p]], 1);
}

__global__ void k_pairs_fill(const int64_t* __restrict__ idx0, const int64_t* __restrict__ idx1,
                             const float* __restrict__ diff, long long P, const int32_t* __restrict__ start,
                             int32_t* __restrict__ cursor, int32_t* __restrict__ csr_j, float4* __restrict__ csr_d) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int a = (int)idx0[p], b = (int)idx1[p];
  // reference convention (neighbors.py:107-111): diff = x[idx0] - x[idx1] + shift
  const float dx = diff[3 * p], dy = diff[3 * p + 1], dz = diff[3 * p + 2];
  const float R = sqrtf(dx * dx + dy * dy + dz * dz);
  const int sa = start[a] + atomicAdd(&cursor[a], 1);
  csr_j[sa] = b;
  csr_d[sa] = make_float4(-dx, -dy, -dz, R);  // seen from a: neighbour b sits at r_b - r_a = -diff
  const int sb = start[b] + atomicAdd(&cursor[b], 1);
  csr_j[sb] = a;
  csr_d[sb] = make_float4(dx, dy, dz, R);
}

__global__ void k_row_overflow(const int32_t* __restrict__ start, int n, int cap, int32_t* __restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && start[i + 1] - start[i] > cap) atomicOr(status, ANI_STATUS_NBR_OVERFLOW);
}


// ---- full neighbour list with ghost atoms (LAMMPS / pmemd style) -> per-atom rows -------------------
// ilist[g] = a local atom, its numneigh[g] neighbours follow each other in jlist (built by the MD engine with
// cutoff + skin, ghost atoms are ordinary entries of coords at their image positions): screen with the true
// cutoff and compact (csrc/aev.cu:1048-1126 postProcessNbrList2 of the reference).  Thread per local atom.
template <bool FILL>
__global__ void k_full_list_rows(const float* __restrict__ coords, const int32_t* __restrict__ ilist,
                                 const int32_t* __restrict__ jstart, const int32_t* __restrict__ jlist, int n_i,
                                 int n_all, float rcr, int32_t* __restrict__ counts,
                                 const int32_t* __restrict__ row_start, int32_t* __restrict__ row_j,
                                 float4* __restrict__ row_d) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_i) return;
  const int i = ilist[g];
  if (i < 0 || i >= n_all) return;
  const float xi = coords[3 * i], yi = coords[3 * i + 1], zi = coords[3 * i + 2];
  const float r2c = rcr * rcr;
  int out = FILL ? row_start[i] : 0, cnt = 0;
  for (int e = jstart[g]; e < jstart[g + 1]; ++e) {
    const int j = jlist[e];
    if (j < 0 || j >= n_all || j == i) continue;
    const float dx = coords[3 * j] - xi, dy = coords[3 * j + 1] - yi, dz = coords[3 * j + 2] - zi;
    const float r2 = dx * dx + dy * dy + dz * dz;
    if (r2 > r2c) continue;
    if (FILL) {
      row_j[out] = j;
      row_d[out] = make_float4(dx, dy, dz, sqrtf(r2));
      ++out;
    }
    ++cnt;
  }
  if (!FILL) counts[i] = cnt;
}

// phase trace of k_aev_forward_cta: only the "aevtrace" build variant records it
extern "C" int ani_b200_debug_aev_trace(long long* buf) {
#if ANI_AEV_FWD_TRACE
  if (cudaMemcpyToSymbol(g_aev_fwd_trace, &buf, sizeof(buf)) != cudaSuccess) return ANI_ERR_CUDA;
  return ANI_OK;
#else
  (void)buf;
  return ANI_ERR_UNSUPPORTED;
#endif
}

}  // namespace ani

using namespace ani;

extern "C" int ani_b200_aev_forward(const ani_aev_params* params, const ani_grid* grid, const int32_t* bin_start,
                                    const float* spos, const int32_t* sbin, const float* bucket_ranges,
                                    const int32_t* bucket_species, const int32_t* species_mask, int n, int lo, int hi,
                                    const int32_t* row_of,
                                    float* aev, int ldx, int layout, int32_t* nbr_cnt, int32_t* nbr_list,
                                    int nbr_cap, int32_t* status, void* stream) {
  int rc = check_params(params);
  if (rc != ANI_OK) return rc;
  if (!bin_start || !sbin || !nbr_cnt || !nbr_list) return ANI_ERR_BAD_ARG;
  // (the species offsets are addressed through the bucket ids stored in the range records)
  return launch_aev_forward(params, grid, bin_start, spos, sbin, bucket_ranges, bucket_ranges ? bucket_species : nullptr,
                            species_mask, ExplicitNbrs{nullptr, nullptr, nullptr}, n, lo, hi, row_of, aev, ldx, layout, nbr_cnt,
                            nbr_list, nbr_cap, status, stream);
}

extern "C" int ani_b200_aev_backward(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                                     const int32_t* sorted_orig, const int32_t* species_mask, int n, int lo, int hi,
                                     const int32_t* row_of, const float* grad_aev, int ldx, const int32_t* nbr_cnt,
                                     const int32_t* nbr_list, int nbr_cap, float* grad_coords, int32_t* status,
                                     int max_elements, double* virial, void* stream) {
  int rc = check_params(params);
  if (rc != ANI_OK) return rc;
  if (!nbr_cnt || !nbr_list) return ANI_ERR_BAD_ARG;
  return launch_aev_backward(params, grid, spos, sorted_orig, n, lo, hi, row_of, grad_aev, ldx, nbr_cnt, nbr_list,
                             ExplicitNbrs{nullptr, nullptr, nullptr}, species_mask, nbr_cap, grad_coords, status,
                             stream, max_elements, virial);
}

// grid mode 3 (ani_b200_prepare_step_cells): the same kernels, image shifts from the lattice table
extern "C" int ani_b200_aev_forward_cells(const ani_aev_params* params, const ani_grid* grid, const int32_t* bin_start,
                                          const float* spos, const int32_t* sbin, const float* bucket_ranges,
                                          const int32_t* bucket_species, const int32_t* species_mask, int n, int lo,
                                          int hi, const int32_t* row_of, float* aev, int ldx, int layout,
                                          int32_t* nbr_cnt, int32_t* nbr_list, int nbr_cap, int32_t* status,
                                          const float* lattice, void* stream) {
  int rc = check_params(params);
  if (rc != ANI_OK) return rc;
  if (!bin_start || !sbin || !nbr_cnt || !nbr_list || !lattice) return ANI_ERR_BAD_ARG;
  return launch_aev_forward(params, grid, bin_start, spos, sbin, bucket_ranges, bucket_ranges ? bucket_species : nullptr,
                            species_mask, ExplicitNbrs{nullptr, nullptr, nullptr}, n, lo, hi, row_of, aev, ldx, layout, nbr_cnt,
                            nbr_list, nbr_cap, status, stream, lattice);
}

extern "C" int ani_b200_aev_backward_cells(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                                           const int32_t* sorted_orig, const int32_t* species_mask, int n, int lo, int hi,
                                           const int32_t* row_of, const float* grad_aev, int ldx, const int32_t* nbr_cnt,
                                           const int32_t* nbr_list, int nbr_cap, float* grad_coords, int32_t* status,
                                           int max_elements, double* virial, const float* lattice, void* stream) {
  int rc = check_params(params);
  if (rc != ANI_OK) return rc;
  if (!nbr_cnt || !nbr_list || !lattice) return ANI_ERR_BAD_ARG;
  return launch_aev_backward(params, grid, spos, sorted_orig, n, lo, hi, row_of, grad_aev, ldx, nbr_cnt, nbr_list,
                             ExplicitNbrs{nullptr, nullptr, nullptr}, species_mask, nbr_cap, grad_coords, status,
                             stream, max_elements, virial, lattice);
}

extern "C" int ani_b200_aev_backward_members(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                                             const int32_t* sorted_orig, const int32_t* species_mask, int n, int lo,
                                             int hi, const int32_t* row_of, const float* grad_slabs, int ldx,
                                             long long slab_stride, const int32_t* members, int n_members,
                                             const int32_t* nbr_cnt, const int32_t* nbr_list, int nbr_cap,
                                             float* grad_members, int32_t* status, int max_elements, void* stream) {
  return launch_aev_backward_members(params, grid, spos, sorted_orig, species_mask, n, lo, hi, row_of, grad_slabs, ldx,
                                     slab_stride, members, n_members, nbr_cnt, nbr_list, nbr_cap, grad_members, status,
                                     max_elements, nullptr, stream);
}

extern "C" int ani_b200_aev_backward_members_cells(const ani_aev_params* params, const ani_grid* grid,
                                                   const float* spos, const int32_t* sorted_orig,
                                                   const int32_t* species_mask, int n, int lo, int hi,
                                                   const int32_t* row_of, const float* grad_slabs, int ldx,
                                                   long long slab_stride, const int32_t* members, int n_members,
                                                   const int32_t* nbr_cnt, const int32_t* nbr_list, int nbr_cap,
                                                   float* grad_members, int32_t* status, int max_elements,
                                                   const float* lattice, void* stream) {
  if (!lattice) return ANI_ERR_BAD_ARG;
  return launch_aev_backward_members(params, grid, spos, sorted_orig, species_mask, n, lo, hi, row_of, grad_slabs, ldx,
                                     slab_stride, members, n_members, nbr_cnt, nbr_list, nbr_cap, grad_members, status,
                                     max_elements, lattice, stream);
}

extern "C" int ani_b200_pairs_to_rows(const int64_t* idx0, const int64_t* idx1, const float* diff_vectors,
                                      int64_t num_pairs, int n, int nbr_cap, int32_t* row_start, int32_t* row_j,
                                      float* row_d, int32_t* scratch_i32, int32_t* status, void* stream) {
  if (!row_start || !row_j || !row_d || !scratch_i32 || !status || n < 1 || num_pairs < 0) return ANI_ERR_BAD_ARG;
  if (num_pairs > 0 && (!idx0 || !idx1 || !diff_vectors)) return ANI_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* counts = scratch_i32;            // [n]
  int32_t* cursor = scratch_i32 + n;        // [n]
  cudaMemsetAsync(scratch_i32, 0, sizeof(int32_t) * 2 * (size_t)n, st);
  const int pb = (int)((num_pairs + 255) / 256);
  if (num_pairs > 0) k_pairs_count<<<pb, 256, 0, st>>>(idx0, idx1, (long long)num_pairs, counts);
  k_scan_i32<<<1, 1024, 0, st>>>(counts, n, row_start);
  if (num_pairs > 0)
    k_pairs_fill<<<pb, 256, 0, st>>>(idx0, idx1, diff_vectors, (long long)num_pairs, row_start, cursor, row_j,
                                     reinterpret_cast<float4*>(row_d));
  k_row_overflow<<<(n + 255) / 256, 256, 0, st>>>(row_start, n, nbr_cap, status);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_full_nbrlist_to_rows(const float* coords, int n_all, const int32_t* ilist,
                                             const int32_t* numneigh, const int32_t* jlist, int n_i, float cutoff,
                                             int nbr_cap, int32_t* row_start, int32_t* row_j, float* row_d,
                                             int32_t* scratch_i32, int32_t* status, void* stream) {
  if (!coords || !row_start || !row_j || !row_d || !scratch_i32 || !status || n_all < 1 || n_i < 0 || cutoff <= 0.f)
    return ANI_ERR_BAD_ARG;
  if (n_i > 0 && (!ilist || !numneigh || !jlist)) return ANI_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* counts = scratch_i32;               // [n_all]
  int32_t* jstart = scratch_i32 + n_all;       // [n_i + 1]
  cudaMemsetAsync(counts, 0, sizeof(int32_t) * (size_t)n_all, st);
  k_scan_i32<<<1, 1024, 0, st>>>(numneigh, n_i, jstart);
  const int nb = (n_i + 127) / 128;
  if (n_i > 0)
    k_full_list_rows<false><<<nb, 128, 0, st>>>(coords, ilist, jstart, jlist, n_i, n_all, cutoff, counts, nullptr,
                                                nullptr, nullptr);
  k_scan_i32<<<1, 1024, 0, st>>>(counts, n_all, row_start);
  if (n_i > 0)
    k_full_list_rows<true><<<nb, 128, 0, st>>>(coords, ilist, jstart, jlist, n_i, n_all, cutoff, nullptr, row_start,
                                               row_j, reinterpret_cast<float4*>(row_d));
  k_row_overflow<<<(n_all + 255) / 256, 256, 0, st>>>(row_start, n_all, nbr_cap, status);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_aev_forward_rows(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                                         const int32_t* row_start, const int32_t* row_j, const float* row_d, int n,
                                         const int32_t* row_of, float* aev, int ldx, int layout, int nbr_cap,
                                         int32_t* status, void* stream) {
  if (!row_start || !row_j || !row_d) return ANI_ERR_BAD_ARG;
  return launch_aev_forward(params, grid, nullptr, spos, nullptr, nullptr, nullptr, nullptr,
                            ExplicitNbrs{row_start, row_j, reinterpret_cast<const float4*>(row_d)}, n, 0, n, row_of,
                            aev, ldx, layout, nullptr, nullptr, nbr_cap, status, stream);
}

extern "C" int ani_b200_aev_backward_rows(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                                          const int32_t* sorted_orig, const int32_t* row_start, const int32_t* row_j,
                                          const float* row_d, int n, const int32_t* row_of, const float* grad_aev,
                                          int ldx, int nbr_cap, float* grad_coords, int32_t* status, void* stream) {
  if (!row_start || !row_j || !row_d) return ANI_ERR_BAD_ARG;
  return launch_aev_backward(params, grid, spos, sorted_orig, n, 0, n, row_of, grad_aev, ldx, nullptr, nullptr,
                             ExplicitNbrs{row_start, row_j, reinterpret_cast<const float4*>(row_d)}, nullptr,
                             nbr_cap, grad_coords, status, stream);
}

extern "C" int ani_b200_half_neighbor_count(const ani_grid* grid, const int32_t* bin_start, const float* spos,
                                            const int32_t* sbin, const int32_t* sorted_orig, int n, float cutoff,
                                            int32_t* pair_start, void* stream) {
  if (!grid || !bin_start || !spos || !sbin || !sorted_orig || !pair_start || n < 1) return ANI_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  // counts go to pair_start[n+1 .. 2n], the scan to pair_start[0 .. n]
  int32_t* counts = pair_start + (n + 1);
  k_half_list<false><<<(n + 127) / 128, 128, 0, st>>>(grid, bin_start, reinterpret_cast<const float4*>(spos), sbin,
                                                      sorted_orig, n, cutoff, counts, nullptr, 0, nullptr, nullptr,
                                                      nullptr, nullptr, nullptr);
  k_scan_i32<<<1, 1024, 0, st>>>(counts, n, pair_start);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_half_neighbor_fill(const ani_grid* grid, const int32_t* bin_start, const float* spos,
                                           const int32_t* sbin, const int32_t* sorted_orig, int n, float cutoff,
                                           const int32_t* pair_start, int64_t cap, int64_t* idx0, int64_t* idx1,
                                           float* distances, float* diff_vectors, int32_t* status, void* stream) {
  if (!grid || !bin_start || !spos || !sbin || !sorted_orig || !pair_start || !idx0 || !idx1 || !distances ||
      !diff_vectors || !status || n < 1)
    return ANI_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  k_half_list<true><<<(n + 127) / 128, 128, 0, st>>>(grid, bin_start, reinterpret_cast<const float4*>(spos), sbin,
                                                     sorted_orig, n, cutoff, nullptr, pair_start, (long long)cap,
                                                     idx0, idx1, distances, diff_vectors, status);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}
