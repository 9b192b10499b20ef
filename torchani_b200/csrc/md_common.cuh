// Pieces shared by the device loops of md.cu (MD integrators), opt.cu (FIRE) and neb.cu (NEB under FIRE): the float64
// cell determinant and inverse, the float32 coordinates of a master position wrapped into the cell, the fixed-shape
// block tree their per-block partial sums go through, and FIRE's scalar update.
#pragma once
#include "common.cuh"

namespace ani {

// determinant of the cell rows m
__device__ __forceinline__ double det3(const double* m) {
  return m[0] * (m[4] * m[8] - m[5] * m[7]) + m[1] * (m[5] * m[6] - m[3] * m[8]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// inverse of the cell rows m (frac = r @ inv)
__device__ __forceinline__ void invert3(const double* m, double* inv) {
  const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
  const double det = m[0] * c00 + m[1] * c01 + m[2] * c02;
  const double r = 1.0 / det;
  inv[0] = c00 * r;
  inv[1] = (m[2] * m[7] - m[1] * m[8]) * r;
  inv[2] = (m[1] * m[5] - m[2] * m[4]) * r;
  inv[3] = c01 * r;
  inv[4] = (m[0] * m[8] - m[2] * m[6]) * r;
  inv[5] = (m[2] * m[3] - m[0] * m[5]) * r;
  inv[6] = c02 * r;
  inv[7] = (m[1] * m[6] - m[0] * m[7]) * r;
  inv[8] = (m[0] * m[4] - m[1] * m[3]) * r;
}

// float64 cell rows and inverse of conformer c (f32 rows at cells + c * stride; nullptr = open), by thread 0 into
// shared memory
__device__ __forceinline__ void load_cell(const float* cells, int stride, int c, double* cell, double* inv) {
  if (threadIdx.x == 0 && cells) {
    const float* f = cells + (size_t)c * stride;
    for (int k = 0; k < 9; ++k) cell[k] = (double)f[k];
    invert3(cell, inv);
  }
}

// float32 coordinates of master position x of atom i: wrapped into the cell (fractional coordinates minus their floor)
// when periodic, so that the float32 copy never holds a far-away image
__device__ __forceinline__ void write_coords(float* coords, size_t i, double x, double y, double z, bool periodic,
                                             const double* cell, const double* inv) {
  if (periodic) {
    const double f0 = floor(x * inv[0] + y * inv[3] + z * inv[6]);
    const double f1 = floor(x * inv[1] + y * inv[4] + z * inv[7]);
    const double f2 = floor(x * inv[2] + y * inv[5] + z * inv[8]);
    x -= f0 * cell[0] + f1 * cell[3] + f2 * cell[6];
    y -= f0 * cell[1] + f1 * cell[4] + f2 * cell[7];
    z -= f0 * cell[2] + f1 * cell[5] + f2 * cell[8];
  }
  coords[3 * i + 0] = (float)x;
  coords[3 * i + 1] = (float)y;
  coords[3 * i + 2] = (float)z;
}

// fixed-shape tree over the block (blockDim.x == ANI_MD_BLOCK): the sums of v[0..NS), the max of w; thread 0 gets the
// results.  sv holds NS * ANI_MD_BLOCK doubles, sw ANI_MD_BLOCK.
template <int NS>
__device__ __forceinline__ void block_reduce(double* v, double& w, double* sv, double* sw) {
#pragma unroll
  for (int k = 0; k < NS; ++k) sv[k * ANI_MD_BLOCK + threadIdx.x] = v[k];
  sw[threadIdx.x] = w;
  __syncthreads();
#pragma unroll
  for (int s = ANI_MD_BLOCK / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
#pragma unroll
      for (int k = 0; k < NS; ++k) sv[k * ANI_MD_BLOCK + threadIdx.x] += sv[k * ANI_MD_BLOCK + threadIdx.x + s];
      sw[threadIdx.x] = fmax(sw[threadIdx.x], sw[threadIdx.x + s]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < NS; ++k) v[k] = sv[k * ANI_MD_BLOCK];
  w = sw[0];
}

// FIRE's scalar update of optimisation c (a conformer of opt.cu, a band of neb.cu) at step t from the totals
// {P, F2, V2, max |f_i|^2}, by thread 0 of every block of the optimisation (the same inputs, so the same results
// everywhere): mix = {c1, c2 + dt, dt * min(1, maxstep / |dr|), frozen}.  The leader block (one per optimisation)
// writes the record {t, *energy, fmax} of step t (rows of RECORD words), the convergence step and the scalars of step
// t + 1, and the leader of optimisation 0 the step counter.
template <int RECORD>
__device__ inline void fire_scalars(const ani_opt_state& s, int c, long long t, const double* tot, bool leader,
                                    const double* energy, double* mix) {
  const double* par = s.params + (size_t)c * ANI_OPT_PARAMS;   // dt0, maxstep, dtmax, Nmin, finc, fdec, astart, fa, fmax
  const double* sc = s.scalars + ((size_t)(t & 1) * s.n_conf + c) * ANI_OPT_SCALARS;
  const double p = tot[0], f2 = tot[1], v2 = tot[2], fmax_ = sqrt(tot[3]);
  double dt = sc[0], al = sc[1], n = sc[2];
  // conv_step[c] is written below by the leader block of this optimisation only, and only with the value t: a block
  // that reads it concurrently sees -1 or t, and "converged before this step" is false for both
  const long long cs = s.conv_step[c];
  const bool before = cs >= 0 && cs < t;
  const bool conv = !before && fmax_ < par[8];
  const bool frozen = before || conv;
  double c1 = 1.0, c2 = 0.0;   // t = 0: v' = v + dt f, and dt is not shrunk
  if (!frozen && t > 0) {
    if (p > 0.0) {
      c1 = 1.0 - al;
      c2 = al * sqrt(v2 / f2);
      if (n > par[3]) {
        dt = fmin(dt * par[4], par[2]);
        al *= par[7];
      }
      n += 1.0;
    } else {
      c1 = 0.0;
      al = par[6];
      dt *= par[5];
      n = 0.0;
    }
  }
  const double cf = c2 + dt;
  const double dr = dt * sqrt(c1 * c1 * v2 + 2.0 * c1 * cf * p + cf * cf * f2);   // |dt v'|: every term is >= 0
  mix[0] = c1;
  mix[1] = cf;
  mix[2] = dt * (dr > par[1] ? par[1] / dr : 1.0);
  mix[3] = frozen ? 1.0 : 0.0;
  if (!leader) return;
  double* nx = s.scalars + ((size_t)((t + 1) & 1) * s.n_conf + c) * ANI_OPT_SCALARS;
  nx[0] = dt;
  nx[1] = al;
  nx[2] = n;
  double* row = s.record + ((size_t)(t % s.record_rows) * s.n_conf + c) * RECORD;
  row[0] = (double)t;
  row[1] = *energy;
  row[2] = fmax_;
  if (conv) s.conv_step[c] = t;
  if (c == 0) s.counter[0] = t + 1;
}

}  // namespace ani
