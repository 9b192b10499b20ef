// Query-by-committee statistics of an ensemble step (arch.py:439-576 of the reference): from the per-member gradients
// of ani_b200_aev_backward_members and the per-member atomic energies of ani_b200_reduce_energies, the ensemble-mean
// gradient, per atom the mean, relative stdev and relative range of the members' force magnitudes, and per conformer
// the members' energies in float64 and the energy QBC factor.  Two small launches, no atomics: every output is written
// by exactly one thread, so the results are deterministic.
#include "terms.cuh"

namespace ani {

// ---- query-by-committee statistics of the members' forces and energies ----------------------------------------------
struct QbcArgs {
  const float* grad_members;   // [count][n][3]
  const float* member_atomic;  // [M][n]
  const int32_t* species;      // [n]
  const double* sae;           // [S] or nullptr
  float* grad;                 // [n][3]
  float* atom_stats;           // [3][n]
  double* member_energies;     // [count][n_conf]
  double* qbc;                 // [n_conf]
  int n, n_conf, n_per_conf;
  ActiveMembers ms;            // output k of grad_members / member_energies is member ms.idx[k]
};

// one thread per atom: the mean gradient and the statistics of the members' force magnitudes (arch.py:543-576)
__global__ void __launch_bounds__(256) k_qbc_atoms(const __grid_constant__ QbcArgs q) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= q.n) return;
  const float eps = 1e-8f;
  float gx = 0.f, gy = 0.f, gz = 0.f, sum = 0.f, mx = -1.f, mn = 3.0e38f;
  float mag[ANI_MAX_MEMBERS];
#pragma unroll
  for (int k = 0; k < ANI_MAX_MEMBERS; ++k) {
    mag[k] = 0.f;
    if (k < q.ms.count) {
      const float* g = q.grad_members + ((size_t)k * q.n + a) * 3;
      const float x = g[0], y = g[1], z = g[2];
      gx += x;
      gy += y;
      gz += z;
      mag[k] = sqrtf(x * x + y * y + z * z);
      sum += mag[k];
      mx = fmaxf(mx, mag[k]);
      mn = fminf(mn, mag[k]);
    }
  }
  const float inv = 1.0f / (float)q.ms.count;
  q.grad[3 * (size_t)a + 0] = gx * inv;
  q.grad[3 * (size_t)a + 1] = gy * inv;
  q.grad[3 * (size_t)a + 2] = gz * inv;
  const float mean = sum * inv;
  float rstd = 0.f, rrange = 1.f;  // one member: stdev 0, range 1
  if (q.ms.count > 1) {
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < ANI_MAX_MEMBERS; ++k)
      if (k < q.ms.count) ss += (mag[k] - mean) * (mag[k] - mean);
    const float sd = sqrtf(ss / (float)(q.ms.count - 1));  // unbiased
    rstd = (sd + eps) / (mean + eps);
    rrange = ((mx - mn) + eps) / (mean + eps);
  }
  q.atom_stats[a] = mean;
  q.atom_stats[(size_t)q.n + a] = rstd;
  q.atom_stats[2 * (size_t)q.n + a] = rrange;
}

// one CTA per conformer: member energies in float64 and qbc = std_m(E_m) / sqrt(real atoms) (arch.py:439-485)
__global__ void __launch_bounds__(256) k_qbc_conformers(const __grid_constant__ QbcArgs q) {
  __shared__ double red[ANI_MAX_MEMBERS + 1][8];
  const int c = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double e[ANI_MAX_MEMBERS + 1];  // per member, then the number of real atoms
#pragma unroll
  for (int k = 0; k <= ANI_MAX_MEMBERS; ++k) e[k] = 0.0;
  for (int t = threadIdx.x; t < q.n_per_conf; t += blockDim.x) {
    const int a = c * q.n_per_conf + t;
    const int sp = q.species[a];
    if (sp < 0) continue;
    const double self = q.sae ? q.sae[sp] : 0.0;
#pragma unroll
    for (int k = 0; k < ANI_MAX_MEMBERS; ++k)
      if (k < q.ms.count) e[k] += (double)q.member_atomic[(size_t)q.ms.idx[k] * q.n + a] + self;
    e[ANI_MAX_MEMBERS] += 1.0;
  }
#pragma unroll
  for (int k = 0; k <= ANI_MAX_MEMBERS; ++k) {
    double v = e[k];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(ANI_FULL_MASK, v, o);
    if (lane == 0) red[k][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double em[ANI_MAX_MEMBERS + 1];
  for (int k = 0; k <= ANI_MAX_MEMBERS; ++k) {
    em[k] = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) em[k] += red[k][w];
  }
  double mean = 0.0;
  for (int k = 0; k < q.ms.count; ++k) {
    q.member_energies[(size_t)k * q.n_conf + c] = em[k];
    mean += em[k];
  }
  mean /= q.ms.count;
  double sd = 0.0;
  if (q.ms.count > 1) {
    double ss = 0.0;
    for (int k = 0; k < q.ms.count; ++k) ss += (em[k] - mean) * (em[k] - mean);
    sd = sqrt(ss / (q.ms.count - 1));
  }
  q.qbc[c] = sd / sqrt(em[ANI_MAX_MEMBERS]);
}

}  // namespace ani

using namespace ani;

extern "C" int ani_b200_ensemble_qbc(const float* grad_members, const int32_t* members, int n_members,
                                     const float* member_atomic, const int32_t* species, const double* sae, int n_conf,
                                     int n_per_conf, float* grad, float* atom_stats, double* member_energies,
                                     double* qbc, void* stream) {
  if (!grad_members || !members || !member_atomic || !species || !grad || !atom_stats || !member_energies || !qbc)
    return ANI_ERR_BAD_ARG;
  if (n_members < 1 || n_conf < 1 || n_per_conf < 1) return ANI_ERR_BAD_ARG;
  QbcArgs q;
  const int rc = active_members(members, n_members, q.ms);
  if (rc != ANI_OK) return rc;
  q.grad_members = grad_members;
  q.member_atomic = member_atomic;
  q.species = species;
  q.sae = sae;
  q.grad = grad;
  q.atom_stats = atom_stats;
  q.member_energies = member_energies;
  q.qbc = qbc;
  q.n = n_conf * n_per_conf;
  q.n_conf = n_conf;
  q.n_per_conf = n_per_conf;
  cudaStream_t st = (cudaStream_t)stream;
  k_qbc_atoms<<<(q.n + 255) / 256, 256, 0, st>>>(q);
  k_qbc_conformers<<<n_conf, 256, 0, st>>>(q);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}
