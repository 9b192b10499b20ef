// Pair potentials evaluated over the neighbour list of the step, or over a neighbour search of their own cutoff.
//
// The AEV forward leaves, for every processed atom, the neighbours within Rcr as words (sorted index | image code
// << 26), BOTH directions of every pair.  A pair potential with a cutoff <= Rcr therefore needs no neighbour search of
// its own: the warp that owns atom i walks i's words, rebuilds Delta_ij = r_j + shift - r_i exactly as the AEV backward
// does (image_shift of common.cuh, in the lattice of the central atom's conformer in grid mode 3) and sums
//   e_i      = 1/2 sum_j E(R_ij) fc(R_ij)                 (potentials/core.py:196-200, the atomic split)
//   dE/dr_i  = sum_j d[E fc]/dR (-Delta_ij / R_ij)        (the whole gradient on i: the list is full)
//   W_ab    += 1/2 sum_j (d[E fc]/dR Delta_a / R) Delta_b (the "f dot r" virial of ase.py:164-168)
// No scatter and no atomics on the forces, a fixed summation order (lane-strided partial sums, butterfly reduction),
// and central-atom shards need nothing new: an atom's gradient comes from the rank that owns it, a pair's energy is
// split between the owners of its two ends.
//
// Functional forms (potentials/xtb.py:57-77, potentials/zbl.py:68-81, potentials/lj.py:118-145,
// potentials/fixed_coulomb.py:28-81), d = max(R, 1e-7) * to_bohr (to_bohr = 1 for the LJ kinds, which work in A):
//   0 xTB           E = y_ab / d * exp(-sqrt_alpha_ab * d^k_ab)
//   1 ZBL           E = Z_a Z_b / d * sum_q c_q exp(-x_q * d * (Z_a^p + Z_b^p) / k)
//   2 LennardJones  E = 4 eps_ab (x^12 - x^6), x = sigma_ab / d
//   3 RepulsionLJ   E = 4 eps_ab x^12
//   4 DispersionLJ  E = -4 eps_ab x^6
//   5 FixedCoulomb  E = qq_ab / d                         (qq_ab = q_a q_b / dielectric)
//   6 FixedMNOK     E = qq_ab / sqrt(d^2 + inv_eta_ab^2), d = R * to_bohr without the clamp
// Arithmetic: expf / sqrtf / powf and true divisions (the repulsion is of order 1 Ha at 0.4 A, so the approximate MUFU
// forms of the AEV kernels would cost the 1e-5 relative bar on atomic energies); d^1.5 is d * sqrt(d).
//
// Kinds 0 and 1 run over the AEV's neighbour words (k_pair_potential, cutoff <= Rcr).  Every kind also runs over
// search_neighbours of terms.cuh at its own cutoff (k_pair_potential_search): the LJ and Coulomb terms are used at
// 8-12 A or without a cutoff, far beyond Rcr.
#include "terms.cuh"

namespace ani {

constexpr int PAIR_WARPS = 8;

// E and dE/dd of each kind at d (Bohr, or A for the LJ kinds)
__device__ __forceinline__ float pair_xtb(const ani_pair_params& P, int a, int b, float d, float& dE) {
  const float y = P.a[a][b], sa = P.b[a][b], k = P.c[a][b];
  const float dk = (k == 1.5f) ? d * sqrtf(d) : (k == 1.0f) ? d : powf(d, k);
  const float E = y / d * expf(-sa * dk);
  dE = -E * (1.0f + sa * k * dk) / d;
  return E;
}

__device__ __forceinline__ float pair_zbl(const ani_pair_params& P, int a, int b, float d, float& dE) {
  const float zz = P.a[a][b], s = P.b[a][b];
  float sum = 0.f, dsum = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float t = P.screen_coeff[q] * expf(-P.screen_exp[q] * s * d);
    sum += t;
    dsum = fmaf(-P.screen_exp[q] * s, t, dsum);
  }
  const float E = zz / d * sum;
  dE = (zz * dsum - E) / d;
  return E;
}

__device__ __forceinline__ float pair_lj(const ani_pair_params& P, int a, int b, float d, float& dE) {
  const float x = P.b[a][b] / d, x2 = x * x, x6 = x2 * x2 * x2, x12 = x6 * x6;
  const float e4 = 4.f * P.a[a][b];
  dE = e4 * (6.f * x6 - 12.f * x12) / d;
  return e4 * (x12 - x6);
}

__device__ __forceinline__ float pair_lj_repulsion(const ani_pair_params& P, int a, int b, float d, float& dE) {
  const float x = P.b[a][b] / d, x2 = x * x, x6 = x2 * x2 * x2;
  const float E = 4.f * P.a[a][b] * (x6 * x6);
  dE = -12.f * E / d;
  return E;
}

__device__ __forceinline__ float pair_lj_dispersion(const ani_pair_params& P, int a, int b, float d, float& dE) {
  const float x = P.b[a][b] / d, x2 = x * x, x6 = x2 * x2 * x2;
  const float E = -4.f * P.a[a][b] * x6;
  dE = -6.f * E / d;
  return E;
}

__device__ __forceinline__ float pair_coulomb(const ani_pair_params& P, int a, int b, float d, float& dE) {
  const float E = P.a[a][b] / d;
  dE = -E / d;
  return E;
}

__device__ __forceinline__ float pair_mnok(const ani_pair_params& P, int a, int b, float d, float& dE) {
  const float ie = P.b[a][b];
  const float u = fmaf(d, d, ie * ie);
  const float E = P.a[a][b] / sqrtf(u);
  dE = -E * d / u;
  return E;
}

// E(R) fc(R) and its derivative with respect to R (Angstrom) for the element pair (a, b)
__device__ __forceinline__ void pair_energy(const ani_pair_params& P, int a, int b, float R, float& e, float& de) {
  const bool clamp = P.kind != 6;                // potentials/core.py:137-139; FixedMNOK does not clamp
  const float d = (clamp ? fmaxf(R, 1e-7f) : R) * P.to_bohr;
  float E, dE;                                   // dE: dE/dd
  switch (P.kind) {
    case 0: E = pair_xtb(P, a, b, d, dE); break;
    case 1: E = pair_zbl(P, a, b, d, dE); break;
    case 2: E = pair_lj(P, a, b, d, dE); break;
    case 3: E = pair_lj_repulsion(P, a, b, d, dE); break;
    case 4: E = pair_lj_dispersion(P, a, b, d, dE); break;
    case 5: E = pair_coulomb(P, a, b, d, dE); break;
    default: E = pair_mnok(P, a, b, d, dE); break;
  }
  dE = (!clamp || R >= 1e-7f) ? dE * P.to_bohr : 0.f;   // the clamp has no slope below its floor
  float f = 1.f, df = 0.f;
  if (P.cutoff_fn != 2) cutoff_value_grad(R, P.cutoff, P.cutoff_fn, f, df);
  e = E * f;
  de = fmaf(dE, f, E * df);
}

// One warp per sorted atom i in lo..hi-1.  Everything is ADDED to what the step has produced so far (the AEV
// backward's atomics into grad, the energy reduction's stores into atomic / member_atomic / energies), by
// add_atom_term and add_conformer_energies of terms.cuh.
template <bool LAT, bool VIRIAL>
__global__ void __launch_bounds__(PAIR_WARPS * 32)
    k_pair_potential(const __grid_constant__ ani_pair_params P, const ani_grid* __restrict__ grid,
                     const float4* __restrict__ spos, const int32_t* __restrict__ sorted_orig, int n, int lo, int hi,
                     int n_per_conf, const int32_t* __restrict__ nbr_cnt, const int32_t* __restrict__ nbr_list, int cap,
                     const float* __restrict__ lattice, const __grid_constant__ TermOut out,
                     const __grid_constant__ ActiveMembers ms) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const ani_grid g = *grid;
  hi = min(hi, g.n_real);
  const int i = lo + blockIdx.x * PAIR_WARPS + warp;
  int conf_out = -1;
  float e_out = 0.f;
  if (i < hi) {
    const float4 pi = spos[i];
    const int si = __float_as_int(pi.w);
    const int oi = sorted_orig[i];
    const int conf_i = oi / n_per_conf;   // the neighbours of an atom lie in its conformer
    const int cnt = min(nbr_cnt[i], cap);
    float e = 0.f, gx = 0.f, gy = 0.f, gz = 0.f;
    float vir[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) vir[k] = 0.f;
    for (int t = lane; t < cnt && si >= 0; t += 32) {
      const int word = nbr_list[(size_t)i * cap + t];
      const int j = word & ANI_IDX_MASK;
      const int code = (unsigned)word >> ANI_IMG_SHIFT;
      const float4 p = spos[j];
      float3 sh = make_float3(0.f, 0.f, 0.f);
      if (code != 13) sh = LAT ? image_shift(lattice, conf_i, code) : image_shift(g, code);
      const float dx = (p.x + sh.x) - pi.x, dy = (p.y + sh.y) - pi.y, dz = (p.z + sh.z) - pi.z;
      const float R = sqrtf(dx * dx + dy * dy + dz * dz);
      if (P.cutoff_fn != 2 && R > P.cutoff) continue;
      float ep, de;
      pair_energy(P, si, __float_as_int(p.w), R, ep, de);
      e = fmaf(0.5f, ep, e);
      const float sc = R >= 1e-7f ? de / R : 0.f;   // dE/dDelta = sc * Delta
      const float fx = sc * dx, fy = sc * dy, fz = sc * dz;
      gx -= fx;
      gy -= fy;
      gz -= fz;
      if (VIRIAL) add_outer(vir, fx, fy, fz, dx, dy, dz);
    }
    if (si >= 0) {
      e_out = add_atom_term<true, VIRIAL>(out, ms, n, g.mode, oi, conf_i, e, gx, gy, gz, vir);
      conf_out = conf_i;
    }
  }
  add_conformer_energies<PAIR_WARPS>(out.energies, e_out, conf_out);
}

// The same sums over search_neighbours at the potential's own cutoff (cutoff_fn 2: no cutoff, open systems only): one
// warp per owned sorted atom, both directions of every pair, outputs and ordering rules of k_pair_potential.  A periodic
// width below cutoff + skin ORs ANI_STATUS_CELL_TOO_SMALL and the atom writes nothing.
template <bool LAT, bool VIRIAL>
__global__ void __launch_bounds__(PAIR_WARPS * 32)
    k_pair_potential_search(const __grid_constant__ ani_pair_params P, const ani_grid* __restrict__ grid,
                            const int32_t* __restrict__ bin_start, const float4* __restrict__ spos,
                            const int32_t* __restrict__ sorted_orig, int n, int lo, int hi, int n_per_conf, float skin,
                            const float* __restrict__ lattice, const __grid_constant__ TermOut out,
                            const __grid_constant__ ActiveMembers ms, int32_t* __restrict__ status) {
  __shared__ SearchHit s_q[PAIR_WARPS][SEARCH_QUEUE];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const ani_grid g = *grid;
  hi = min(hi, g.n_real);
  const int i = lo + blockIdx.x * PAIR_WARPS + warp;
  const float cutoff = P.cutoff_fn == 2 ? INFINITY : P.cutoff;
  int conf_out = -1;
  float e_out = 0.f;
  if (i < hi) {
    const float4 pi = spos[i];
    const int si = __float_as_int(pi.w);
    const int oi = sorted_orig[i];
    const int conf_i = oi / n_per_conf;
    float e = 0.f, gx = 0.f, gy = 0.f, gz = 0.f;
    float vir[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) vir[k] = 0.f;
    if (si >= 0) {
      const bool ok = search_neighbours<LAT>(cutoff, g, bin_start, spos, lattice, i, pi, conf_i, skin, s_q[warp],
                                             [&](int j, int sj, float dx, float dy, float dz, float R) {
        if (sj < 0) return;
        float ep, de;
        pair_energy(P, si, sj, R, ep, de);
        e = fmaf(0.5f, ep, e);
        const float sc = R >= 1e-7f ? de / R : 0.f;   // dE/dDelta = sc * Delta
        const float fx = sc * dx, fy = sc * dy, fz = sc * dz;
        gx -= fx;
        gy -= fy;
        gz -= fz;
        if (VIRIAL) add_outer(vir, fx, fy, fz, dx, dy, dz);
      });
      if (!ok) {
        if (lane == 0 && status) atomicOr(status, ANI_STATUS_CELL_TOO_SMALL);
      } else {
        e_out = add_atom_term<true, VIRIAL>(out, ms, n, g.mode, oi, conf_i, e, gx, gy, gz, vir);
        conf_out = conf_i;
      }
    }
  }
  add_conformer_energies<PAIR_WARPS>(out.energies, e_out, conf_out);
}

// The same potential over a caller-supplied HALF pair list (the reference's Neighbors tuple; diff = x[idx0] - x[idx1] +
// shift): one thread per pair, float atomics (not the hot path).  Pairs that touch a ghost atom count half
// (potentials/core.py:170-177); pairs beyond the cutoff and pairs with a padding atom contribute nothing.
__global__ void k_pair_potential_pairs(const __grid_constant__ ani_pair_params P, const int32_t* __restrict__ species,
                                       const int64_t* __restrict__ idx0, const int64_t* __restrict__ idx1,
                                       const float* __restrict__ distances, const float* __restrict__ diff,
                                       const uint8_t* __restrict__ ghost, long long num_pairs, int n_per_conf,
                                       float* __restrict__ atomic, double* __restrict__ energies,
                                       float* __restrict__ grad) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= num_pairs) return;
  const long long i0 = idx0[p], i1 = idx1[p];
  const int s0 = species[i0], s1 = species[i1];
  const float R = distances[p];
  if (s0 < 0 || s1 < 0 || (P.cutoff_fn != 2 && R > P.cutoff)) return;
  float e, de;
  pair_energy(P, s0, s1, R, e, de);
  if (ghost && (ghost[i0] | ghost[i1])) {
    e *= 0.5f;
    de *= 0.5f;
  }
  add_pair_energy(atomic, energies, i0, i1, n_per_conf, e);
  if (grad) add_pair_grad(grad, diff, p, i0, i1, R >= 1e-7f ? de / R : 0.f);
}

static int check_pair_params(const ani_pair_params* p) {
  const int rc = check_term_params(p);
  if (rc != ANI_OK) return rc;
  return p->kind >= 0 && p->kind <= 6 ? ANI_OK : ANI_ERR_BAD_ARG;
}

static int launch_pair_potential(const ani_pair_params* params, const ani_grid* grid, const float* spos,
                                 const int32_t* sorted_orig, int n, int lo, int hi, int n_conf, int n_per_conf,
                                 const int32_t* nbr_cnt, const int32_t* nbr_list, int nbr_cap, float* atomic,
                                 double* energies, float* grad_coords, double* virial, float* member_atomic,
                                 float* grad_members, const int32_t* members, int n_members, const float* lattice,
                                 bool want_lattice, void* stream) {
  int rc = check_pair_params(params);
  if (rc != ANI_OK) return rc;
  ActiveMembers ms;
  rc = check_step_term_args(grid, spos, sorted_orig, n, lo, hi, n_conf, n_per_conf, lattice, want_lattice,
                            member_atomic, grad_members, members, n_members, ms);
  if (rc != ANI_OK) return rc;
  if (!nbr_cnt || !nbr_list || nbr_cap < 1) return ANI_ERR_BAD_ARG;
  if (hi == lo) return ANI_OK;
  const int blocks = (hi - lo + PAIR_WARPS - 1) / PAIR_WARPS;
  const TermOut out{atomic, energies, grad_coords, virial, member_atomic, grad_members};
  auto launch = [&](auto kernel) {
    kernel<<<blocks, PAIR_WARPS * 32, 0, (cudaStream_t)stream>>>(
        *params, grid, reinterpret_cast<const float4*>(spos), sorted_orig, n, lo, hi, n_per_conf, nbr_cnt, nbr_list,
        nbr_cap, lattice, out, ms);
  };
  if (want_lattice) {
    virial ? launch(k_pair_potential<true, true>) : launch(k_pair_potential<true, false>);
  } else {
    virial ? launch(k_pair_potential<false, true>) : launch(k_pair_potential<false, false>);
  }
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

static int launch_pair_potential_search(const ani_pair_params* params, const ani_grid* grid, const int32_t* bin_start,
                                        const float* spos, const int32_t* sorted_orig, int n, int lo, int hi,
                                        int n_conf, int n_per_conf, float skin, float* atomic, double* energies,
                                        float* grad_coords, double* virial, float* member_atomic, float* grad_members,
                                        const int32_t* members, int n_members, int32_t* status, const float* lattice,
                                        bool want_lattice, void* stream) {
  int rc = check_pair_params(params);
  if (rc != ANI_OK) return rc;
  ActiveMembers ms;
  rc = check_step_term_args(grid, spos, sorted_orig, n, lo, hi, n_conf, n_per_conf, lattice, want_lattice,
                            member_atomic, grad_members, members, n_members, ms);
  if (rc != ANI_OK) return rc;
  if (!bin_start || !(skin >= 0.f)) return ANI_ERR_BAD_ARG;
  if (hi == lo) return ANI_OK;
  const int blocks = (hi - lo + PAIR_WARPS - 1) / PAIR_WARPS;
  const TermOut out{atomic, energies, grad_coords, virial, member_atomic, grad_members};
  auto launch = [&](auto kernel) {
    kernel<<<blocks, PAIR_WARPS * 32, 0, (cudaStream_t)stream>>>(
        *params, grid, bin_start, reinterpret_cast<const float4*>(spos), sorted_orig, n, lo, hi, n_per_conf, skin,
        lattice, out, ms, status);
  };
  if (want_lattice) {
    virial ? launch(k_pair_potential_search<true, true>) : launch(k_pair_potential_search<true, false>);
  } else {
    virial ? launch(k_pair_potential_search<false, true>) : launch(k_pair_potential_search<false, false>);
  }
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

}  // namespace ani

extern "C" int ani_b200_pair_potential(const ani_pair_params* params, const ani_grid* grid, const float* spos,
                                       const int32_t* sorted_orig, int n, int lo, int hi, int n_conf, int n_per_conf,
                                       const int32_t* nbr_cnt, const int32_t* nbr_list, int nbr_cap, float* atomic,
                                       double* energies, float* grad_coords, double* virial, float* member_atomic,
                                       float* grad_members, const int32_t* members, int n_members, void* stream) {
  return ani::launch_pair_potential(params, grid, spos, sorted_orig, n, lo, hi, n_conf, n_per_conf, nbr_cnt, nbr_list,
                                    nbr_cap, atomic, energies, grad_coords, virial, member_atomic, grad_members,
                                    members, n_members, nullptr, false, stream);
}

extern "C" int ani_b200_pair_potential_cells(const ani_pair_params* params, const ani_grid* grid, const float* spos,
                                             const int32_t* sorted_orig, int n, int lo, int hi, int n_conf,
                                             int n_per_conf, const int32_t* nbr_cnt, const int32_t* nbr_list,
                                             int nbr_cap, float* atomic, double* energies, float* grad_coords,
                                             double* virial, float* member_atomic, float* grad_members,
                                             const int32_t* members, int n_members, const float* lattice,
                                             void* stream) {
  return ani::launch_pair_potential(params, grid, spos, sorted_orig, n, lo, hi, n_conf, n_per_conf, nbr_cnt, nbr_list,
                                    nbr_cap, atomic, energies, grad_coords, virial, member_atomic, grad_members,
                                    members, n_members, lattice, true, stream);
}

extern "C" int ani_b200_pair_potential_search(const ani_pair_params* params, const ani_grid* grid,
                                              const int32_t* bin_start, const float* spos, const int32_t* sorted_orig,
                                              int n, int lo, int hi, int n_conf, int n_per_conf, float skin,
                                              float* atomic, double* energies, float* grad_coords, double* virial,
                                              float* member_atomic, float* grad_members, const int32_t* members,
                                              int n_members, int32_t* status, void* stream) {
  return ani::launch_pair_potential_search(params, grid, bin_start, spos, sorted_orig, n, lo, hi, n_conf, n_per_conf,
                                           skin, atomic, energies, grad_coords, virial, member_atomic, grad_members,
                                           members, n_members, status, nullptr, false, stream);
}

extern "C" int ani_b200_pair_potential_search_cells(const ani_pair_params* params, const ani_grid* grid,
                                                    const int32_t* bin_start, const float* spos,
                                                    const int32_t* sorted_orig, int n, int lo, int hi, int n_conf,
                                                    int n_per_conf, float skin, float* atomic, double* energies,
                                                    float* grad_coords, double* virial, float* member_atomic,
                                                    float* grad_members, const int32_t* members, int n_members,
                                                    int32_t* status, const float* lattice, void* stream) {
  return ani::launch_pair_potential_search(params, grid, bin_start, spos, sorted_orig, n, lo, hi, n_conf, n_per_conf,
                                           skin, atomic, energies, grad_coords, virial, member_atomic, grad_members,
                                           members, n_members, status, lattice, true, stream);
}

extern "C" int ani_b200_pair_potential_pairs(const ani_pair_params* params, const int32_t* species,
                                             const int64_t* idx0, const int64_t* idx1, const float* distances,
                                             const float* diff_vectors, const uint8_t* ghost_flags, int64_t num_pairs,
                                             int n_conf, int n_per_conf, float* atomic, double* energies,
                                             float* grad_coords, void* stream) {
  const int rc = ani::check_pair_params(params);
  if (rc != ANI_OK) return rc;
  if (num_pairs < 0 || n_conf < 1 || n_per_conf < 1) return ANI_ERR_BAD_ARG;
  if (num_pairs == 0) return ANI_OK;
  if (!species || !idx0 || !idx1 || !distances) return ANI_ERR_BAD_ARG;
  if (grad_coords && !diff_vectors) return ANI_ERR_BAD_ARG;
  const long long blocks = (num_pairs + 255) / 256;
  if (blocks > 0x7fffffffLL) return ANI_ERR_BAD_ARG;
  ani::k_pair_potential_pairs<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      *params, species, idx0, idx1, distances, diff_vectors, ghost_flags, num_pairs, n_per_conf, atomic, energies,
      grad_coords);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}
