// Pieces shared by the device loops of md.cu (MD integrators), opt.cu (FIRE, cell FIRE), lbfgs.cu (L-BFGS) and neb.cu
// (NEB under FIRE):
//   host      the arguments every loop launch takes (LoopArgs), the cell_mode decoding of the init entry points and the
//             launch-shape check of the step entry points
//   device    the float64 cell determinant and inverse; the float32 coordinates of a master position wrapped into the
//             cell, and of a whole conformer (the tail of the one-CTA-per-conformer init kernels); the fixed-shape
//             block tree and the ordered warp reduction their per-block partials go through; FIRE's scalar reset,
//             scalar update and move
#pragma once
#include "common.cuh"

namespace ani {

// what every loop launch takes besides its state
struct LoopArgs {
  const float* grad;          // f32[n][3] dE/dx (Hartree / A), input order
  const double* energies;     // f64[n_conf]
  const float* cells;         // cell rows (f32[9]) of conformer c at cells + c * cell_stride; nullptr = open
  int cell_stride;
  float* coords;              // f32[n][3]
  int reset;                  // the init entry point's flag (ani_b200_md_init: the centre-of-mass momentum removal)
};

// the cells of an init entry point's cell_mode (0 open, 1 one cell, 2 one per conformer) into a; false when invalid
inline bool init_cells(LoopArgs& a, const float* cells, int cell_mode) {
  if (cell_mode < 0 || cell_mode > 2 || (cell_mode && !cells)) return false;
  a.cells = cell_mode ? cells : nullptr;
  a.cell_stride = cell_mode == 2 ? 9 : 0;
  return true;
}

// a step launch over (blocks of a conformer's atoms) x conformers: n_conf * n_per_conf atoms must fit an int and
// n_conf the grid's y (or z) extent
inline int launch_shape(long long n_conf, long long n_per_conf) {
  return n_conf * n_per_conf > 0x7fffffffLL || n_conf > 65535 ? ANI_ERR_UNSUPPORTED : ANI_OK;
}

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

// the float32 coordinates of the master positions x of conformer c (A atoms), wrapped into its cell: the tail of the
// one-CTA-per-conformer init kernels, after their own writes to x
__device__ __forceinline__ void conformer_coords(const LoopArgs& a, int c, int A, const double* x) {
  __shared__ double cell[9], inv[9];
  load_cell(a.cells, a.cell_stride, c, cell, inv);
  __syncthreads();
  for (int j = threadIdx.x; j < A; j += blockDim.x) {
    const size_t i = (size_t)c * A + j;
    write_coords(a.coords, i, x[3 * i + 0], x[3 * i + 1], x[3 * i + 2], a.cells, cell, inv);
  }
}

// the fixed shuffle tree towards lane 0 over a warp: the sums of v[0..NS), the maxima of v[NS..NS+NM)
template <int NS, int NM>
__device__ __forceinline__ void warp_tree(double* v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int k = 0; k < NS + NM; ++k) {
      const double u = __shfl_down_sync(ANI_FULL_MASK, v[k], o);
      v[k] = k < NS ? v[k] + u : fmax(v[k], u);
    }
}

// the ordered reduction of n partials by one warp (lane = the thread's lane): lane l sums (and takes maxima of)
// partials l, l + 32, ... in order, then warp_tree; lane 0 gets the totals.  part(b, v) writes partial b's NS summed
// and then NM maximised values to v.
template <int NS, int NM, class Part>
__device__ __forceinline__ void warp_reduce(int lane, int n, Part part, double* tot) {
#pragma unroll
  for (int k = 0; k < NS + NM; ++k) tot[k] = 0.0;
  for (int b = lane; b < n; b += ANI_WARP) {
    double v[NS + NM];
    part(b, v);
#pragma unroll
    for (int k = 0; k < NS + NM; ++k) tot[k] = k < NS ? tot[k] + v[k] : fmax(tot[k], v[k]);
  }
  warp_tree<NS, NM>(tot);
}

// warp_reduce of n FIRE partials {P, F2, V2, max |f_i|^2} at p (4 words each)
__device__ __forceinline__ void fire_totals(const double* p, int n, double* tot) {
  warp_reduce<3, 1>(threadIdx.x, n, [&](int b, double* v) {
    for (int k = 0; k < 4; ++k) v[k] = p[4 * (unsigned)b + k];
  }, tot);
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

// FIRE's scalars {dt0, astart, 0} of optimisation c at the parity slot of step t
__device__ __forceinline__ void fire_reset(const ani_opt_state& s, int c, long long t) {
  const double* par = s.params + (size_t)c * ANI_OPT_PARAMS;
  double* sc = s.scalars + ((size_t)(t & 1) * s.n_conf + c) * ANI_OPT_SCALARS;
  sc[0] = par[0];
  sc[1] = par[6];
  sc[2] = 0.0;
}

// FIRE's move of one atom with force f by mix (fire_scalars): v' = c1 v + (c2 + dt) f, x += st v'; returns x(t+1) in xn
__device__ __forceinline__ void fire_move(const double* mix, const double* f, double* v, double* x, double* xn) {
  const double c1 = mix[0], cf = mix[1], st = mix[2];
  const double vx = c1 * v[0] + cf * f[0], vy = c1 * v[1] + cf * f[1], vz = c1 * v[2] + cf * f[2];
  xn[0] = x[0] + st * vx;
  xn[1] = x[1] + st * vy;
  xn[2] = x[2] + st * vz;
  v[0] = vx;
  v[1] = vy;
  v[2] = vz;
  x[0] = xn[0];
  x[1] = xn[1];
  x[2] = xn[2];
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
