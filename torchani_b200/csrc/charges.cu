// Atomic charges and dipoles of charge models (ANIq, ANImbis): the normaliser and dipole of the reference
// (electro.py:29-156, ChargeNormalizer.forward and DipoleComputer.forward) on the raw per-row outputs of a charge
// network pass.
//
// Per conformer, with e_i the element of atom i (-1 = padding) and q_raw_i its raw charge:
//   w_i = W[e_i] (* q_raw_i^2 with scale_by_q2), 0 for padding
//   q_i = q_raw_i + (Q - sum_j q_raw_j) w_i / sum_j w_j            (normalize; else q_i = q_raw_i)
//   mu  = sum_i q_i (r_i - r_ref)   over the real atoms, r_ref = centre of mass / of geometry / origin
// mu is formed as sum_i q_i r_i - (sum_i q_i) r_ref, with the stored (float32) q_i.
//
// One CTA per conformer walks the conformer's atoms with a block-strided loop, twice: pass 1 sums q_raw, w and the
// reference-frame moments, pass 2 writes q_i and sums q_i r_i and q_i.  Every sum is float64, accumulated per thread
// in increasing atom order and reduced across the block by a fixed butterfly / warp order: no atomics, so repeated
// runs give identical bits.  The block size follows the conformer size (64 threads for small molecules, 1024 for a
// 10 k-atom system), so that a batch of hundreds of small conformers and one large system take the same path.
#include "common.cuh"

namespace ani {

constexpr int CHG_SUMS = 6;   // doubles per block reduction
constexpr int CHG_UNROLL = 4; // independent atoms in flight per thread (the raw charges are a three-level gather)

struct ChargeArgs {
  const float* q_raw;           // rows (with row_of / orig_to_sorted) or input order
  const int32_t* row_of;
  const int32_t* orig_to_sorted;
  const int32_t* species;
  const float* coords;          // f32[n][3], input order
  int n_per_conf, num_species;
  int scale_by_q2, normalize, frame;
  double total_charge;
  float weights[ANI_MAX_SPECIES];
  float masses[ANI_MAX_SPECIES];
  float* charges;               // f32[n]
  double* dipoles;              // f64[n_conf][3] or nullptr
};

// sum of CHG_SUMS doubles over the block in a fixed order; every thread gets the totals
__device__ __forceinline__ void block_sum(double (&v)[CHG_SUMS], double (*red)[CHG_SUMS]) {
#pragma unroll
  for (int k = 0; k < CHG_SUMS; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(ANI_FULL_MASK, v[k], o);
  const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();   // (red is reused by the second reduction)
  if (lane_id() == 0)
#pragma unroll
    for (int k = 0; k < CHG_SUMS; ++k) red[warp][k] = v[k];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < CHG_SUMS; ++k) {
    double s = 0.0;
    for (int w = 0; w < nw; ++w) s += red[w][k];
    v[k] = s;
  }
}

__device__ __forceinline__ float raw_charge(const ChargeArgs& a, int i, int e) {
  if (e < 0) return 0.f;
  if (!a.row_of) return a.q_raw[i];
  return a.q_raw[a.row_of[a.orig_to_sorted[i]]];
}

__global__ void __launch_bounds__(1024) k_charges(const __grid_constant__ ChargeArgs a) {
  __shared__ double red[32][CHG_SUMS];
  const int A = a.n_per_conf;
  const long long base = (long long)blockIdx.x * A;
  const bool want_dipole = a.dipoles != nullptr;
  // pass 1: sum q_raw, sum w, and the reference-frame moments (mass or count, and its first moment)
  double s[CHG_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int j0 = threadIdx.x; j0 < A; j0 += CHG_UNROLL * blockDim.x) {
    int e[CHG_UNROLL];
    float q[CHG_UNROLL];
#pragma unroll
    for (int u = 0; u < CHG_UNROLL; ++u) {
      const int j = j0 + u * blockDim.x;
      e[u] = j < A ? a.species[base + j] : -1;
    }
#pragma unroll
    for (int u = 0; u < CHG_UNROLL; ++u) q[u] = raw_charge(a, (int)(base + j0 + u * blockDim.x), e[u]);
#pragma unroll
    for (int u = 0; u < CHG_UNROLL; ++u) {
      if (e[u] < 0) continue;
      const long long i = base + j0 + u * blockDim.x;
      s[0] += (double)q[u];
      double w = (double)a.weights[e[u]];
      if (a.scale_by_q2) w *= (double)q[u] * (double)q[u];
      s[1] += w;
      if (want_dipole && a.frame != 2) {
        const double m = a.frame == 0 ? (double)a.masses[e[u]] : 1.0;
        s[2] += m;
        s[3] += m * (double)a.coords[3 * i];
        s[4] += m * (double)a.coords[3 * i + 1];
        s[5] += m * (double)a.coords[3 * i + 2];
      }
    }
  }
  block_sum(s, red);
  const double excess = a.total_charge - s[0];
  const double inv_w = 1.0 / s[1];
  double ref[3] = {0.0, 0.0, 0.0};
  if (a.frame != 2 && s[2] != 0.0)
#pragma unroll
    for (int d = 0; d < 3; ++d) ref[d] = s[3 + d] / s[2];
  // pass 2: q_i, and sum q_i r_i, sum q_i
  double t[CHG_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int j0 = threadIdx.x; j0 < A; j0 += CHG_UNROLL * blockDim.x) {
    int e[CHG_UNROLL];
    float q[CHG_UNROLL];
#pragma unroll
    for (int u = 0; u < CHG_UNROLL; ++u) {
      const int j = j0 + u * blockDim.x;
      e[u] = j < A ? a.species[base + j] : -1;
    }
#pragma unroll
    for (int u = 0; u < CHG_UNROLL; ++u) q[u] = raw_charge(a, (int)(base + j0 + u * blockDim.x), e[u]);
#pragma unroll
    for (int u = 0; u < CHG_UNROLL; ++u) {
      const int j = j0 + u * blockDim.x;
      if (j >= A) continue;
      const long long i = base + j;
      float qi = 0.f;
      if (e[u] >= 0) {
        qi = q[u];
        if (a.normalize) {
          double w = (double)a.weights[e[u]];
          if (a.scale_by_q2) w *= (double)q[u] * (double)q[u];
          qi = (float)((double)q[u] + excess * (w * inv_w));
        }
        if (want_dipole) {
          t[0] += (double)qi * (double)a.coords[3 * i];
          t[1] += (double)qi * (double)a.coords[3 * i + 1];
          t[2] += (double)qi * (double)a.coords[3 * i + 2];
          t[3] += (double)qi;
        }
      }
      a.charges[i] = qi;
    }
  }
  if (!want_dipole) return;
  block_sum(t, red);
  if (threadIdx.x == 0)
#pragma unroll
    for (int d = 0; d < 3; ++d) a.dipoles[3 * blockIdx.x + d] = t[d] - t[3] * ref[d];
}

}  // namespace ani

extern "C" int ani_b200_charges(const float* q_raw, const int32_t* row_of, const int32_t* orig_to_sorted,
                                const int32_t* species, const float* coords, int n_conf, int n_per_conf,
                                const float* weights, int num_species, int scale_by_q2, int normalize,
                                double total_charge, const float* masses, int frame, float* charges_out,
                                double* dipoles_out, void* stream) {
  if (!q_raw || !species || !charges_out || (!row_of != !orig_to_sorted)) return ANI_ERR_BAD_ARG;
  if (n_conf < 1 || n_per_conf < 1 || num_species < 1 || num_species > ANI_MAX_SPECIES) return ANI_ERR_BAD_ARG;
  if (frame < 0 || frame > 2) return ANI_ERR_BAD_ARG;
  if (normalize && !weights) return ANI_ERR_BAD_ARG;
  if (dipoles_out && (!coords || (frame == 0 && !masses))) return ANI_ERR_BAD_ARG;
  ani::ChargeArgs a;
  a.q_raw = q_raw;
  a.row_of = row_of;
  a.orig_to_sorted = orig_to_sorted;
  a.species = species;
  a.coords = coords;
  a.n_per_conf = n_per_conf;
  a.num_species = num_species;
  a.scale_by_q2 = scale_by_q2 != 0;
  a.normalize = normalize != 0;
  a.frame = frame;
  a.total_charge = total_charge;
  for (int s = 0; s < ANI_MAX_SPECIES; ++s) {
    a.weights[s] = (weights && s < num_species) ? weights[s] : 0.f;
    a.masses[s] = (masses && s < num_species) ? masses[s] : 0.f;
  }
  a.charges = charges_out;
  a.dipoles = dipoles_out;
  // block size: the conformer's atoms in one strided pass of CHG_UNROLL per thread where possible, 64..1024 threads
  int threads = 64;
  while (threads < 1024 && threads * ani::CHG_UNROLL < n_per_conf) threads *= 2;
  ani::k_charges<<<n_conf, threads, 0, (cudaStream_t)stream>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}
