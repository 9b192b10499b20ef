// D3(BJ) two-body dispersion (potentials/dftd3.py:140-311, TwoBodyDispersionD3) inside the fused step.
//
// With d = R * to_bohr, a = s_i, b = s_j and every pair within the cutoff:
//   CN_i   = sum_j 1 / (1 + exp(-k1 (k2 (rcov_a + rcov_b) / d - 1)))           (no envelope, dftd3.py:251-272)
//   L_pq   = exp(-k3 ((CN_i - CNa_pq)^2 + (CN_j - CNb_pq)^2)), 0 where C6ref_pq <= 0
//   C6_ij  = (sum_pq C6ref_pq L_pq + eps) / (sum_pq L_pq + eps), eps = 1e-35        (dftd3.py:274-311)
//   E_ij   = -(s6 C6 / (d^6 + damp6_ab) + s8 3 C6 sqrt_q_ab / (d^8 + damp8_ab)) fc(R)   (dftd3.py:221-246)
// with damp_n = (a1 R0_ab + a2)^n (BeckeJohnsonDamp, dftd3.py:102-110).  The atomic split gives half of E_ij to each
// end (potentials/core.py:196-200).  Forces have a direct part (C6 fixed) and the coordination-number chain
//   dE/dr_i += sum_j (dE/dCN_i + dE/dCN_j) count'(R_ij) dR_ij/dr_i,   dE/dCN_i = sum_j dE_ij/dC6_ij dC6_ij/dCN_i.
//
// Two numerical rules of this implementation:
//   * Exponent scaling.  Both sums of the C6 interpolation are multiplied by exp(k3 g_min), the inverse of their
//     largest Gaussian, so the largest term is exactly 1 and no term underflows in float32 where it would not in
//     float64.  eps is scaled with them, eps exp(k3 g_min) = exp(k3 g_min + ln eps) (capped at e^80, where the ratio
//     is 1 to float32 precision), so the ratio is the reference's also where sum L is not >> eps: coordination
//     numbers far from every reference value, where the reference's C6 moves towards eps / eps = 1.
//   * No valid reference.  An element pair with no positive C6ref gets C6 = 1 and dC6/dCN = 0, as eps / eps does in
//     the reference.
//
// The neighbour search is search_neighbours of terms.cuh: the AEV's neighbour words end at Rcr, D3 reaches 8 A or
// more.  It needs every periodic width >= cutoff + skin; below that the first launch ORs ANI_STATUS_CELL_TOO_SMALL
// and nothing is written.
//
// Three launches, each over the results of the previous one for ALL real atoms:
//   1. CN of every real atom (plain stores into cn[sorted index]),
//   2. dE/dCN of every real atom (dedcn), and for the owned atoms lo..hi-1 the atomic / conformer / member energies,
//      the direct gradient and the direct virial,
//   3. the chain gradient and virial of the owned atoms.
// One warp per sorted atom walks BOTH directions of every pair: no scatter and no atomics on the forces, a fixed
// summation order (lane-strided partial sums, butterfly reduction), and central-atom shards stay correct because
// passes 1-2 run over all atoms on every rank.  Passes 2 and 3 search again instead of reading a list written by
// pass 1 (DESIGN section 4.6): no capacity, no overflow mode.
// Arithmetic: expf and true divisions, as csrc/pair.cu.
#include "terms.cuh"

namespace ani {

constexpr int D3_WARPS = 8;
constexpr int D3_REFS = 25;   // 5 x 5 reference pairs per element pair
constexpr float D3_LN_EPS = -80.5904782547916f;   // ln(1e-35), the eps of dftd3.py:177

// coordination-number count of a pair and its derivative with respect to R (Angstrom)
__device__ __forceinline__ void d3_count(const ani_d3_params& P, int a, int b, float R, float& c, float& dc) {
  const float d = R * P.to_bohr;
  const float rc = P.rcov[a] + P.rcov[b];
  const float t = expf(-P.k1 * (P.k2 * rc / d - 1.0f));
  c = 1.0f / (1.0f + t);
  dc = -(t * P.k1 * P.k2 * rc / (d * d)) * c * c * P.to_bohr;
}

// C6 of the element pair (a, b) at coordination numbers (cni, cnj) and dC6/dcni; with `dcnj` also dC6/dcnj.
// tab: float4 {C6ref, CNa, CNb, 0} per (a, b, p, q).  Exponent scaling: see the head of this file.
template <bool BOTH>
__device__ __forceinline__ void d3_c6(const ani_d3_params& P, const float4* __restrict__ tab, int a, int b, float cni,
                                      float cnj, float& c6, float& dc6i, float& dc6j) {
  const float4* t = tab + (size_t)(a * P.num_species + b) * D3_REFS;
  float gmin = INFINITY;
#pragma unroll 5
  for (int k = 0; k < D3_REFS; ++k) {
    const float4 v = __ldg(t + k);
    const float u = cni - v.y, w = cnj - v.z;
    if (v.x > 0.f) gmin = fminf(gmin, u * u + w * w);
  }
  if (gmin == INFINITY) {   // no valid reference: eps / eps
    c6 = 1.f;
    dc6i = dc6j = 0.f;
    return;
  }
  float W = 0.f, Z = 0.f, Wi = 0.f, Zi = 0.f, Wj = 0.f, Zj = 0.f;
#pragma unroll 5
  for (int k = 0; k < D3_REFS; ++k) {
    const float4 v = __ldg(t + k);
    if (!(v.x > 0.f)) continue;
    const float u = cni - v.y, w = cnj - v.z;
    const float L = expf(-P.k3 * ((u * u + w * w) - gmin));
    W += L;
    Z = fmaf(v.x, L, Z);
    Wi = fmaf(u, L, Wi);
    Zi = fmaf(v.x * u, L, Zi);
    if (BOTH) {
      Wj = fmaf(w, L, Wj);
      Zj = fmaf(v.x * w, L, Zj);
    }
  }
  const float e = expf(fminf(P.k3 * gmin + D3_LN_EPS, 80.f));   // eps, scaled like the sums
  W += e;
  Z += e;
  c6 = Z / W;
  // d(Z/W)/dcn = (Z' W - Z W') / W^2 with dL/dcni = -2 k3 u L (eps is a constant of the unscaled sums)
  dc6i = -2.f * P.k3 * (Zi - c6 * Wi) / W;
  dc6j = BOTH ? -2.f * P.k3 * (Zj - c6 * Wj) / W : 0.f;
}

// pair energy E_ij fc and its derivatives with respect to R (C6 fixed) and to C6
__device__ __forceinline__ void d3_energy(const ani_d3_params& P, int a, int b, float R, float c6, float& e,
                                          float& de_dr, float& de_dc6) {
  const float d = R * P.to_bohr;
  const float d2 = d * d, d6 = d2 * d2 * d2, d8 = d6 * d2;
  const float den6 = d6 + P.damp6[a][b], den8 = d8 + P.damp8[a][b];
  const float s8q = P.s8 * P.c8_scale[a][b];
  const float per_c6 = -(P.s6 / den6 + s8q / den8);          // E / C6 before the envelope
  const float E = c6 * per_c6;
  // dE/dd = C6 (s6 6 d^5 / den6^2 + s8 q 8 d^7 / den8^2)
  const float dE = c6 * (P.s6 * 6.f * d6 / (d * den6 * den6) + s8q * 8.f * d8 / (d * den8 * den8)) * P.to_bohr;
  float f = 1.f, df = 0.f;
  if (P.cutoff_fn != 2) cutoff_value_grad(R, P.cutoff, P.cutoff_fn, f, df);
  e = E * f;
  de_dr = fmaf(dE, f, E * df);
  de_dc6 = per_c6 * f;
}

// PASS 1: cn of every real atom.  PASS 2: dedcn of every real atom, energies + direct gradient / virial of the owned
// atoms.  PASS 3: chain gradient / virial of the owned atoms.  One warp per sorted atom, first = lo (pass 3) or 0.
template <int PASS, bool LAT, bool VIRIAL>
__global__ void __launch_bounds__(D3_WARPS * 32)
    k_dispersion_d3(const __grid_constant__ ani_d3_params P, const float4* __restrict__ tab,
                    const ani_grid* __restrict__ grid, const int32_t* __restrict__ bin_start,
                    const float4* __restrict__ spos, const int32_t* __restrict__ sorted_orig, int n, int first, int lo,
                    int hi, int n_per_conf, float skin, const float* __restrict__ lattice, float* __restrict__ cn,
                    float* __restrict__ dedcn, const __grid_constant__ TermOut out,
                    const __grid_constant__ ActiveMembers ms, int32_t* __restrict__ status) {
  __shared__ SearchHit s_q[D3_WARPS][SEARCH_QUEUE];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const ani_grid g = *grid;
  const int end = min(PASS == 3 ? hi : n, g.n_real);
  const int i = first + blockIdx.x * D3_WARPS + warp;
  int conf_out = -1;
  float e_out = 0.f;
  if (i < end) {
    const float4 pi = spos[i];
    const int si = __float_as_int(pi.w);
    const int oi = sorted_orig[i];
    const int conf_i = oi / n_per_conf;
    const bool owned = i >= lo && i < hi;
    float acc = 0.f, e = 0.f, gx = 0.f, gy = 0.f, gz = 0.f;
    float vir[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) vir[k] = 0.f;
    const float cni = PASS >= 2 ? cn[i] : 0.f;
    const float dedcn_i = PASS == 3 ? dedcn[i] : 0.f;
    bool ok = true;
    if (si >= 0) {
      ok = search_neighbours<LAT>(P.cutoff, g, bin_start, spos, lattice, i, pi, conf_i, skin, s_q[warp],
                                  [&](int j, int sj, float dx, float dy, float dz, float R) {
        if (sj < 0) return;
        if (PASS == 1) {
          float c, dc;
          d3_count(P, si, sj, R, c, dc);
          acc += c;
          return;
        }
        float sc;   // dE/dDelta = sc * Delta
        if (PASS == 2) {
          float c6, dc6i, dc6j, ep, de_dr, de_dc6;
          d3_c6<false>(P, tab, si, sj, cni, cn[j], c6, dc6i, dc6j);
          d3_energy(P, si, sj, R, c6, ep, de_dr, de_dc6);
          acc = fmaf(de_dc6, dc6i, acc);
          if (!owned) return;
          e = fmaf(0.5f, ep, e);
          sc = de_dr / R;
        } else {
          float c, dc;
          d3_count(P, si, sj, R, c, dc);
          sc = (dedcn_i + dedcn[j]) * dc / R;
        }
        const float fx = sc * dx, fy = sc * dy, fz = sc * dz;
        gx -= fx;
        gy -= fy;
        gz -= fz;
        if (VIRIAL) add_outer(vir, fx, fy, fz, dx, dy, dz);
      });
    }
    if (!ok) {   // periodic width below cutoff + skin: raised once, by the first launch
      if (PASS == 1 && lane == 0 && status) atomicOr(status, ANI_STATUS_CELL_TOO_SMALL);
    } else {
      if (PASS <= 2) {
        acc = warp_sum(acc);
        if (lane == 0) (PASS == 1 ? cn : dedcn)[i] = acc;
      }
      if (PASS >= 2 && owned && si >= 0) {
        e_out = add_atom_term<PASS == 2, VIRIAL>(out, ms, n, g.mode, oi, conf_i, e, gx, gy, gz, vir);
        conf_out = conf_i;
      }
    }
  }
  if (PASS == 2) add_conformer_energies<D3_WARPS>(out.energies, e_out, conf_out);
}

// ---- a caller's HALF pair list (not the hot path): one thread per pair, float atomics ----
// diff = x[idx0] - x[idx1] + shift; a pair touching a ghost atom counts half in the energy (potentials/core.py:170-177)
// and fully in the coordination numbers.
__device__ __forceinline__ bool d3_pair_ok(const ani_d3_params& P, const int32_t* species, long long i0, long long i1,
                                           float R) {
  return species[i0] >= 0 && species[i1] >= 0 && (P.cutoff_fn == 2 || R <= P.cutoff);
}

template <int PASS>
__global__ void k_dispersion_d3_pairs(const __grid_constant__ ani_d3_params P, const float4* __restrict__ tab,
                                      const int32_t* __restrict__ species, const int64_t* __restrict__ idx0,
                                      const int64_t* __restrict__ idx1, const float* __restrict__ distances,
                                      const float* __restrict__ diff, const uint8_t* __restrict__ ghost,
                                      long long num_pairs, int n_per_conf, float* __restrict__ cn,
                                      float* __restrict__ dedcn, float* __restrict__ atomic,
                                      double* __restrict__ energies, float* __restrict__ grad) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= num_pairs) return;
  const long long i0 = idx0[p], i1 = idx1[p];
  const float R = distances[p];
  if (!d3_pair_ok(P, species, i0, i1, R)) return;
  const int s0 = species[i0], s1 = species[i1];
  if (PASS == 1) {
    float c, dc;
    d3_count(P, s0, s1, R, c, dc);
    atomicAdd(&cn[i0], c);
    atomicAdd(&cn[i1], c);
    return;
  }
  float sc;
  if (PASS == 2) {
    float c6, dc60, dc61, e, de_dr, de_dc6;
    d3_c6<true>(P, tab, s0, s1, cn[i0], cn[i1], c6, dc60, dc61);
    d3_energy(P, s0, s1, R, c6, e, de_dr, de_dc6);
    if (ghost && (ghost[i0] | ghost[i1])) {
      e *= 0.5f;
      de_dr *= 0.5f;
      de_dc6 *= 0.5f;
    }
    add_pair_energy(atomic, energies, i0, i1, n_per_conf, e);
    if (!grad) return;
    atomicAdd(&dedcn[i0], de_dc6 * dc60);
    atomicAdd(&dedcn[i1], de_dc6 * dc61);
    sc = de_dr / R;
  } else {
    float c, dc;
    d3_count(P, s0, s1, R, c, dc);
    sc = (dedcn[i0] + dedcn[i1]) * dc / R;
  }
  add_pair_grad(grad, diff, p, i0, i1, sc);   // dR/dx0 = diff / R
}

static int check_d3_params(const ani_d3_params* p, const float* tables) {
  return tables ? check_term_params(p) : ANI_ERR_BAD_ARG;
}

static int launch_dispersion_d3(const ani_d3_params* params, const float* tables, const ani_grid* grid,
                                const int32_t* bin_start, const float* spos, const int32_t* sorted_orig, int n, int lo,
                                int hi, int n_conf, int n_per_conf, float skin, float* cn, float* dedcn,
                                float* atomic, double* energies, float* grad_coords, double* virial,
                                float* member_atomic, float* grad_members, const int32_t* members, int n_members,
                                int32_t* status, const float* lattice, bool want_lattice, void* stream) {
  int rc = check_d3_params(params, tables);
  if (rc != ANI_OK) return rc;
  // the fused step searches its own neighbours: it needs a finite cutoff
  if (params->cutoff_fn == 2) return ANI_ERR_BAD_ARG;
  ActiveMembers ms;
  rc = check_step_term_args(grid, spos, sorted_orig, n, lo, hi, n_conf, n_per_conf, lattice, want_lattice,
                            member_atomic, grad_members, members, n_members, ms);
  if (rc != ANI_OK) return rc;
  if (!bin_start || !cn || !dedcn || !(skin >= 0.f)) return ANI_ERR_BAD_ARG;
  const TermOut out{atomic, energies, grad_coords, virial, member_atomic, grad_members};
  const bool want_grad = grad_coords || grad_members || virial;
  const float4* tab = reinterpret_cast<const float4*>(tables);
  const float4* sp = reinterpret_cast<const float4*>(spos);
  cudaStream_t st = (cudaStream_t)stream;
  const int all_blocks = (n + D3_WARPS - 1) / D3_WARPS;
  const int own_blocks = (hi - lo + D3_WARPS - 1) / D3_WARPS;
  auto launch = [&](auto kernel, int blocks, int first) {
    if (blocks > 0)
      kernel<<<blocks, D3_WARPS * 32, 0, st>>>(*params, tab, grid, bin_start, sp, sorted_orig, n, first, lo, hi,
                                               n_per_conf, skin, lattice, cn, dedcn, out, ms, status);
  };
  // pass 2 also needs the direct gradient only where forces are wanted: out carries NULLs otherwise
  if (want_lattice) {
    launch(k_dispersion_d3<1, true, false>, all_blocks, 0);
    virial ? launch(k_dispersion_d3<2, true, true>, all_blocks, 0) : launch(k_dispersion_d3<2, true, false>, all_blocks, 0);
    if (want_grad)
      virial ? launch(k_dispersion_d3<3, true, true>, own_blocks, lo) : launch(k_dispersion_d3<3, true, false>, own_blocks, lo);
  } else {
    launch(k_dispersion_d3<1, false, false>, all_blocks, 0);
    virial ? launch(k_dispersion_d3<2, false, true>, all_blocks, 0) : launch(k_dispersion_d3<2, false, false>, all_blocks, 0);
    if (want_grad)
      virial ? launch(k_dispersion_d3<3, false, true>, own_blocks, lo) : launch(k_dispersion_d3<3, false, false>, own_blocks, lo);
  }
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

}  // namespace ani

extern "C" int ani_b200_dispersion_d3(const ani_d3_params* params, const float* tables, const ani_grid* grid,
                                      const int32_t* bin_start, const float* spos, const int32_t* sorted_orig, int n,
                                      int lo, int hi, int n_conf, int n_per_conf, float skin, float* cn, float* dedcn,
                                      float* atomic, double* energies, float* grad_coords, double* virial,
                                      float* member_atomic, float* grad_members, const int32_t* members, int n_members,
                                      int32_t* status, void* stream) {
  return ani::launch_dispersion_d3(params, tables, grid, bin_start, spos, sorted_orig, n, lo, hi, n_conf, n_per_conf,
                                   skin, cn, dedcn, atomic, energies, grad_coords, virial, member_atomic, grad_members,
                                   members, n_members, status, nullptr, false, stream);
}

extern "C" int ani_b200_dispersion_d3_cells(const ani_d3_params* params, const float* tables, const ani_grid* grid,
                                            const int32_t* bin_start, const float* spos, const int32_t* sorted_orig,
                                            int n, int lo, int hi, int n_conf, int n_per_conf, float skin, float* cn,
                                            float* dedcn, float* atomic, double* energies, float* grad_coords,
                                            double* virial, float* member_atomic, float* grad_members,
                                            const int32_t* members, int n_members, int32_t* status,
                                            const float* lattice, void* stream) {
  return ani::launch_dispersion_d3(params, tables, grid, bin_start, spos, sorted_orig, n, lo, hi, n_conf, n_per_conf,
                                   skin, cn, dedcn, atomic, energies, grad_coords, virial, member_atomic, grad_members,
                                   members, n_members, status, lattice, true, stream);
}

extern "C" int ani_b200_dispersion_d3_pairs(const ani_d3_params* params, const float* tables, const int32_t* species,
                                            const int64_t* idx0, const int64_t* idx1, const float* distances,
                                            const float* diff_vectors, const uint8_t* ghost_flags, int64_t num_pairs,
                                            int n_conf, int n_per_conf, float* cn, float* dedcn, float* atomic,
                                            double* energies, float* grad_coords, void* stream) {
  const int rc = ani::check_d3_params(params, tables);
  if (rc != ANI_OK) return rc;
  if (num_pairs < 0 || n_conf < 1 || n_per_conf < 1) return ANI_ERR_BAD_ARG;
  if (!cn || (grad_coords && !dedcn)) return ANI_ERR_BAD_ARG;
  const size_t n = (size_t)n_conf * n_per_conf;
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(cn, 0, n * sizeof(float), st);
  if (grad_coords) cudaMemsetAsync(dedcn, 0, n * sizeof(float), st);
  ANI_CUDA_CHECK_LAUNCH();
  // an empty list has no pair arrays to point to (as in ani_b200_pair_potential_pairs)
  if (num_pairs == 0) return ANI_OK;
  if (!species || !idx0 || !idx1 || !distances) return ANI_ERR_BAD_ARG;
  if (grad_coords && !diff_vectors) return ANI_ERR_BAD_ARG;
  const long long blocks = (num_pairs + 255) / 256;
  if (blocks > 0x7fffffffLL) return ANI_ERR_BAD_ARG;
  const float4* tab = reinterpret_cast<const float4*>(tables);
  auto launch = [&](auto kernel) {
    kernel<<<(unsigned)blocks, 256, 0, st>>>(*params, tab, species, idx0, idx1, distances, diff_vectors, ghost_flags,
                                             num_pairs, n_per_conf, cn, dedcn, atomic, energies, grad_coords);
  };
  launch(ani::k_dispersion_d3_pairs<1>);
  launch(ani::k_dispersion_d3_pairs<2>);
  if (grad_coords) launch(ani::k_dispersion_d3_pairs<3>);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}
