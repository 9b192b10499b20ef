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
