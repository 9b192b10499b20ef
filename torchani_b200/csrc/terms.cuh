// Pieces shared by the step terms that add per-atom outputs: the pair potentials (pair.cu), D3 (disp.cu), and the
// active-member table of the query-by-committee launches (aev.cu, qbc.cu).
#pragma once
#include "common.cuh"

namespace ani {

// Active members of a query-by-committee step: output k (grad_members, member energies) belongs to member idx[k]
struct ActiveMembers {
  int count;
  int idx[ANI_MAX_MEMBERS];
};

// ms from a caller's list of n_members (0..ANI_MAX_MEMBERS) member indices, each in [0, ANI_MAX_MEMBERS); the unused
// entries are 0.  A list is needed when n_members > 0.
inline int active_members(const int32_t* members, int n_members, ActiveMembers& ms) {
  if (n_members < 0 || n_members > ANI_MAX_MEMBERS || (n_members > 0 && !members)) return ANI_ERR_BAD_ARG;
  ms.count = n_members;
  for (int k = 0; k < ANI_MAX_MEMBERS; ++k) {
    ms.idx[k] = k < n_members ? members[k] : 0;
    if (ms.idx[k] < 0 || ms.idx[k] >= ANI_MAX_MEMBERS) return ANI_ERR_BAD_ARG;
  }
  return ANI_OK;
}

// The fields ani_pair_params and ani_d3_params share: envelope (0 cosine, 1 smooth, 2 none), element count, length
// unit, and a finite positive cutoff under an envelope
template <class Params>
int check_term_params(const Params* p) {
  if (!p) return ANI_ERR_BAD_ARG;
  if (p->cutoff_fn < 0 || p->cutoff_fn > 2) return ANI_ERR_BAD_ARG;
  if (p->num_species < 1 || p->num_species > ANI_MAX_SPECIES) return ANI_ERR_BAD_ARG;
  if (!(p->to_bohr > 0.f)) return ANI_ERR_BAD_ARG;
  if (p->cutoff_fn != 2 && !(p->cutoff > 0.f && p->cutoff < 1e30f)) return ANI_ERR_BAD_ARG;
  return ANI_OK;
}

// The arguments of a term inside the step (ani_b200_pair_potential, ani_b200_dispersion_d3 and their _cells forms):
// the step's grid and sorted positions, n = n_conf * n_per_conf, the owned range lo..hi, the lattice table of the
// _cells forms, and the member list, which member outputs need.  Fills ms.
inline int check_step_term_args(const ani_grid* grid, const float* spos, const int32_t* sorted_orig, int n, int lo,
                                int hi, int n_conf, int n_per_conf, const float* lattice, bool want_lattice,
                                const float* member_atomic, const float* grad_members, const int32_t* members,
                                int n_members, ActiveMembers& ms) {
  if (!grid || !spos || !sorted_orig) return ANI_ERR_BAD_ARG;
  if (want_lattice && !lattice) return ANI_ERR_BAD_ARG;
  if (n_conf < 1 || n_per_conf < 1 || n != n_conf * n_per_conf) return ANI_ERR_BAD_ARG;
  if (lo < 0 || hi > n || lo > hi) return ANI_ERR_BAD_ARG;
  if ((member_atomic || grad_members) && n_members == 0) return ANI_ERR_BAD_ARG;
  return active_members(members, n_members, ms);
}

// The outputs a term adds to; any may be NULL
struct TermOut {
  float* atomic;
  double* energies;
  float* grad;
  double* virial;
  float* member_atomic;
  float* grad_members;
};

__device__ __forceinline__ void add_outer(float (&vir)[9], float fx, float fy, float fz, float dx, float dy, float dz) {
  vir[0] = fmaf(fx, dx, vir[0]); vir[1] = fmaf(fx, dy, vir[1]); vir[2] = fmaf(fx, dz, vir[2]);
  vir[3] = fmaf(fy, dx, vir[3]); vir[4] = fmaf(fy, dy, vir[4]); vir[5] = fmaf(fy, dz, vir[5]);
  vir[6] = fmaf(fz, dx, vir[6]); vir[7] = fmaf(fz, dy, vir[7]); vir[8] = fmaf(fz, dz, vir[8]);
}

// Adds the term of a real atom (original index oi, conformer conf_i) to the outputs, from the lane partial sums of the
// warp that owns it; returns the atom's energy (the warp sum of e).  The virial takes 1/2 of the summed f (x) Delta
// into the slots of the AEV backward: one set per conformer of a periodic batch (grid modes 2, 3), slot blockIdx.x %
// ANI_VIRIAL_SLOTS.  Everything else is a plain read-modify-write by lane 0: every output element of an atom has
// exactly one writer, and the launch is ordered after the kernels that accumulate into the same buffers.  The
// reference adds its potentials to every member of the ensemble (arch.py:365-378).  ENERGY: add e to the atomic and
// member energies.  Warp-uniform.
template <bool ENERGY, bool VIRIAL>
__device__ __forceinline__ float add_atom_term(const TermOut& out, const ActiveMembers& ms, int n, int mode, int oi,
                                               int conf_i, float e, float gx, float gy, float gz,
                                               const float (&vir)[9]) {
  const int lane = threadIdx.x & 31;
  gx = warp_sum(gx);
  gy = warp_sum(gy);
  gz = warp_sum(gz);
  if (ENERGY) e = warp_sum(e);
  if (VIRIAL) {
    double* slots = out.virial + (size_t)(mode >= 2 ? conf_i : 0) * ANI_VIRIAL_SLOTS * 9;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const float v = warp_sum(vir[k]);
      if (lane == 0) atomicAdd(&slots[(blockIdx.x % ANI_VIRIAL_SLOTS) * 9 + k], 0.5 * (double)v);
    }
  }
  if (lane == 0) {
    if (ENERGY && out.atomic) out.atomic[oi] += e;
    if (out.grad) {
      out.grad[3 * (size_t)oi + 0] += gx;
      out.grad[3 * (size_t)oi + 1] += gy;
      out.grad[3 * (size_t)oi + 2] += gz;
    }
    for (int k = 0; k < ms.count; ++k) {
      if (ENERGY && out.member_atomic) out.member_atomic[(size_t)ms.idx[k] * n + oi] += e;
      if (out.grad_members) {
        float* gm = out.grad_members + ((size_t)k * n + oi) * 3;
        gm[0] += gx;
        gm[1] += gy;
        gm[2] += gz;
      }
    }
  }
  return e;
}

// Adds the energies of a CTA's atoms to energies[conformer]: lane 0 of every warp passes its atom's energy and
// conformer (-1: none).  Sorted atoms are conformer-major in a batch, so thread 0 adds one float64 atomic per run of
// equal conformers.  Called by every thread of the CTA; nothing happens without `energies`.
template <int WARPS>
__device__ __forceinline__ void add_conformer_energies(double* energies, float e, int conf) {
  __shared__ float s_e[WARPS];
  __shared__ int s_conf[WARPS];
  if (!energies) return;
  if ((threadIdx.x & 31) == 0) {
    s_e[threadIdx.x >> 5] = e;
    s_conf[threadIdx.x >> 5] = conf;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int c = -1;
    double acc = 0.0;
    for (int w = 0; w < WARPS; ++w) {
      if (s_conf[w] < 0) continue;
      if (s_conf[w] != c) {
        if (c >= 0) atomicAdd(&energies[c], acc);
        c = s_conf[w];
        acc = 0.0;
      }
      acc += (double)s_e[w];
    }
    if (c >= 0) atomicAdd(&energies[c], acc);
  }
}

// ---- the neighbour search at a term's own cutoff (D3, and the pair potentials of ani_b200_pair_potential_search) ----
// It runs on the bucket grid of the step (bin_start, spos, ani_grid; the lattice table in grid mode 3) with a stencil
// of `reach_d = ceil((cutoff + skin) / bucket width_d)` buckets per lattice direction, bucket width = perpendicular
// width / dims.  Offsets -reach..reach are distinct (bucket, image) pairs, so a neighbour inside the cutoff at two
// images (cells between 1x and 2x the cutoff) counts twice, as the reference's multi-image lists count it.  Image codes
// stay the 27 codes of common.cuh, which needs reach_d <= dims_d, i.e. every periodic width >= cutoff + skin.  Open
// systems clip the stencil to the grid (an infinite cutoff walks the whole grid); grid mode 1 (one bucket per
// conformer) walks the conformer's bucket.

// largest bucket b with bin_start[b] <= i: the bucket of sorted atom i (empty buckets share their start with the next)
__device__ __forceinline__ int bucket_of(const int32_t* __restrict__ bin_start, int nbins, int i) {
  int lo = 0, hi = nbins - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(bin_start + mid) <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// a neighbour inside the cutoff, queued in shared memory until the warp has 32 of them
struct SearchHit {
  int j, sj;
  float dx, dy, dz, R;
};
constexpr int SEARCH_QUEUE = 64;

// Calls f(j, sj, dx, dy, dz, R) for every neighbour j of sorted atom i with R <= cutoff (Delta = r_j + shift - r_i;
// cutoff may be +inf on open systems).  The warp screens 32 candidates at a time (about one in eight is inside an 8 A
// cutoff on a 5 A bucket grid) and queues the hits in `q` (SEARCH_QUEUE entries of this warp's shared memory); f runs
// on 32 queued hits at a time, so the per-pair work runs with all lanes busy.  The order of the hits, and so every
// lane's partial sum, depends only on the grid.  Warp-uniform; returns false (nothing visited) if a periodic width is
// below cutoff + skin.
template <bool LAT, class F>
__device__ __forceinline__ bool search_neighbours(float cutoff, const ani_grid& g,
                                                  const int32_t* __restrict__ bin_start,
                                                  const float4* __restrict__ spos, const float* __restrict__ lattice,
                                                  int i, float4 pi, int conf, float skin, SearchHit* __restrict__ q,
                                                  F&& f) {
  const int lane = threadIdx.x & 31;
  const float cut2 = cutoff * cutoff;
  int qn = 0;   // queued hits (warp-uniform)
  auto drain = [&]() {
    const int m = min(qn, 32);
    if (lane < m) {
      const SearchHit h = q[lane];
      f(h.j, h.sj, h.dx, h.dy, h.dz, h.R);
    }
    __syncwarp();
    if (lane < qn - 32) q[lane] = q[lane + 32];
    __syncwarp();
    qn -= m;
  };
  auto run = [&](int lo, int hi, int code) {
    float3 sh = make_float3(0.f, 0.f, 0.f);
    if (code != 13) sh = LAT ? image_shift(lattice, conf, code) : image_shift(g, code);
    for (int b0 = lo; b0 < hi; b0 += 32) {
      const int j = b0 + lane;
      bool hit = false;
      SearchHit h;
      if (j < hi && !(code == 13 && j == i)) {
        const float4 p = spos[j];
        h.dx = (p.x + sh.x) - pi.x;
        h.dy = (p.y + sh.y) - pi.y;
        h.dz = (p.z + sh.z) - pi.z;
        const float r2 = h.dx * h.dx + h.dy * h.dy + h.dz * h.dz;
        hit = r2 <= cut2;
        h.j = j;
        h.sj = __float_as_int(p.w);
        h.R = sqrtf(r2);
      }
      const unsigned m = __ballot_sync(ANI_FULL_MASK, hit);
      if (hit) q[qn + __popc(m & ((1u << lane) - 1u))] = h;
      __syncwarp();
      qn += __popc(m);
      if (qn >= 32) drain();
    }
  };
  if (!LAT && g.mode == 1) {   // one bucket per conformer
    run(__ldg(bin_start + conf), __ldg(bin_start + conf + 1), 13);
    if (qn > 0) drain();
    return true;
  }
  int ix, iy, iz;
  const int base = bucket_coords(g, bucket_of(bin_start, g.nbins, i), ix, iy, iz);
  const float* inv = LAT ? lattice + (size_t)conf * ANI_LATTICE_STRIDE + 9 : g.inv;
  const float reach_len = cutoff + skin;
  int r[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float perp = 1.0f / sqrtf(inv[d] * inv[d] + inv[3 + d] * inv[3 + d] + inv[6 + d] * inv[6 + d]);
    const float reach = ceilf(reach_len * (float)g.dims[d] / perp);
    r[d] = reach <= (float)g.dims[d] ? (int)reach : g.dims[d] + 1;   // (an infinite reach exceeds every grid)
    if (g.pbc) {
      if (r[d] > g.dims[d]) return false;
    } else {
      r[d] = min(r[d], g.dims[d] - 1);
    }
  }
  const int dx_ = g.dims[0], dy_ = g.dims[1], dz_ = g.dims[2];
  for (int ox = -r[0]; ox <= r[0]; ++ox) {
    int jx = ix + ox, wx = jx < 0 ? -1 : (jx >= dx_ ? 1 : 0);
    if (wx && !g.pbc) continue;
    jx -= wx * dx_;
    for (int oy = -r[1]; oy <= r[1]; ++oy) {
      int jy = iy + oy, wy = jy < 0 ? -1 : (jy >= dy_ ? 1 : 0);
      if (wy && !g.pbc) continue;
      jy -= wy * dy_;
      const int row = base + (jx * dy_ + jy) * dz_;
      // the z run iz-r..iz+r in up to three contiguous pieces, one per image
      for (int wz = -1; wz <= 1; ++wz) {
        if (wz && !g.pbc) continue;
        const int zlo = max(iz - r[2], wz * dz_), zhi = min(iz + r[2], wz * dz_ + dz_ - 1);
        if (zlo > zhi) continue;
        run(__ldg(bin_start + row + zlo - wz * dz_), __ldg(bin_start + row + zhi - wz * dz_ + 1),
            (wx + 1) * 9 + (wy + 1) * 3 + (wz + 1));
      }
    }
  }
  if (qn > 0) drain();
  return true;
}

// ---- a caller's HALF pair list (not the hot path): one thread per pair p = (i0, i1), float atomics ----
// the pair's energy e: half to each end's atomic energy, all of it to the conformer of i0
__device__ __forceinline__ void add_pair_energy(float* atomic, double* energies, long long i0, long long i1,
                                                int n_per_conf, float e) {
  if (atomic) {
    atomicAdd(&atomic[i0], 0.5f * e);
    atomicAdd(&atomic[i1], 0.5f * e);
  }
  if (energies) atomicAdd(&energies[i0 / n_per_conf], (double)e);
}

// the pair's gradient dE/d(diff) = sc * diff, diff = x[i0] - x[i1] + shift: + on i0, - on i1
__device__ __forceinline__ void add_pair_grad(float* grad, const float* diff, long long p, long long i0, long long i1,
                                              float sc) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float f = sc * diff[3 * p + k];
    atomicAdd(&grad[3 * i0 + k], f);
    atomicAdd(&grad[3 * i1 + k], -f);
  }
}

}  // namespace ani
