// Nudged elastic band on the device: ASE's NEB (methods "aseneb" and "improvedtangent", optionally with a climbing
// image) relaxed by ASE's FIRE, one optimisation per band over the rows of its interior images.  The interior images
// of B bands are the B (n - 2) conformers of one force step; the endpoints never enter it.  As in opt.cu, the master
// positions, FIRE velocities and per-band scalars stay in device memory and the launches write the float32
// coordinates of the next force step, so K whole steps (NEB + force step) capture into one CUDA graph.
//
// Every tangent is tau = alpha t- + beta t+, so five dot products per image, {a, b, c, p, q} = {t-.t-, t+.t+, t-.t+,
// F.t-, F.t+}, give every scalar of the projection, and the NEB force is f = F + gamma- t- + gamma+ t+.  One step is
// the force step at x(t) followed by three launches, each over (blocks of NEB_BLOCK atoms) x interior images:
//   k_neb_dots     the block's partial sums {a, b, c, p, q} (a block tree of fixed shape)
//   k_neb_project  every block sums its image's partials in order; thread 0 reads the band's energies, forms imax,
//                  (alpha, beta) and gamma-, gamma+; every thread writes f to neb_force, and the block its FIRE
//                  partials {f.v, f.f, v.v, max |f_i|^2}
//   k_neb_update   every block sums all of its band's FIRE partials (fire_totals, as k_opt_update does) and runs
//                  FIRE's scalar rule (fire_scalars); the band's first block writes the
//                  record {t, E_imax, fmax, imax}, conv_step and the scalars of t + 1; every block moves its atoms with
//                  neb_force and writes their float32 coordinates, wrapped into the cell of its image's conformer
// Race rules: the scalars are double-buffered by step parity; conv_step[b] and the record have one writer, the band's
// leader block; the counter follows md.cu (k_neb_dots copies counter[0] to counter[1], the leader of band 0 writes
// t + 1); neb_force and both partial arrays are written by one launch and read only by later ones.  No atomics: the
// same state and forces give the same bits.
#include "md_common.cuh"

namespace ani {

constexpr int NEB_BLOCK = ANI_MD_BLOCK;

struct NebArgs : LoopArgs {   // energies: f64[B (n - 2)] the interior images' energies
  ani_neb_state s;
  int step;                   // k_neb_dots copies the counter (a step, not ani_b200_neb_project)
};

// F, t- and t+ of atom j of interior conformer ci; returns its force_scale (0: F, t- and t+ are all 0)
__device__ __forceinline__ double neb_vectors(const NebArgs& a, int ci, int j, double* f, double* tm, double* tp) {
  const ani_neb_state& s = a.s;
  const int m = s.n_images - 2, A = s.n_atoms;
  const int b = ci / m, i = ci - b * m + 1;
  const size_t k = (size_t)ci * A + j;
  const double fs = s.fire.force_scale[k];
  const double* x = s.fire.x + 3 * k;
  const double* xm = i == 1 ? s.endpoints + 3 * ((size_t)(2 * b) * A + j) : x - 3 * (size_t)A;
  const double* xp = i == m ? s.endpoints + 3 * ((size_t)(2 * b + 1) * A + j) : x + 3 * (size_t)A;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const bool on = fs != 0.0;
    f[d] = on ? -(double)a.grad[3 * k + d] * fs : 0.0;
    tm[d] = on ? x[d] - xm[d] : 0.0;
    tp[d] = on ? xp[d] - x[d] : 0.0;
  }
  return fs;
}

// imax of band b (1 + the first index of the largest interior energy) and a pointer to E_imax
__device__ __forceinline__ int band_imax(const double* energies, int b, int m, const double** emax) {
  const double* e = energies + (size_t)b * m;
  int r = 0;
  for (int q = 1; q < m; ++q)
    if (e[q] > e[r]) r = q;
  *emax = e + r;
  return r + 1;
}

// gamma-, gamma+ of interior conformer ci from its totals {a, b, c, p, q} (thread 0 of k_neb_project)
__device__ void neb_gammas(const NebArgs& a, int ci, const double* dot, double* g) {
  const ani_neb_state& s = a.s;
  const int m = s.n_images - 2, b = ci / m, i = ci - b * m + 1;
  const double* emax;
  const int imax = band_imax(a.energies, b, m, &emax);
  const double* e = a.energies + (size_t)b * m;   // E_i at e[i - 1]
  const double* ee = s.end_energies + 2 * (size_t)b;
  const double e0 = i == 1 ? ee[0] : e[i - 2], e1 = e[i - 1], e2 = i == m ? ee[1] : e[i];
  const double* k = s.springs + (size_t)b * (m + 1);
  const double km = k[i - 1], kp = k[i];
  const bool climb = s.climb[b] != 0.0 && i == imax;
  double al, be;
  if (s.method == ANI_NEB_ASENEB) {
    al = i < imax ? 0.0 : 1.0;
    be = i > imax ? 0.0 : 1.0;
  } else if (e2 > e1 && e1 > e0) {
    al = 0.0;
    be = 1.0;
  } else if (e2 < e1 && e1 < e0) {
    al = 1.0;
    be = 0.0;
  } else {
    const double dn = fabs(e2 - e1), dp = fabs(e0 - e1);
    const double dmax = fmax(dn, dp), dmin = fmin(dn, dp);
    al = e2 > e0 ? dmin : dmax;
    be = e2 > e0 ? dmax : dmin;
  }
  const double ta = dot[0], tb = dot[1], tc = dot[2], p = dot[3], q = dot[4];
  const double ft = al * p + be * q;                                        // F.tau
  // tau.tau, rounded term by term (no contraction into FMAs): t+ = -t- and alpha = beta give exactly 0, as tau is
  const double tt = __dadd_rn(__dadd_rn(__dmul_rn(al * al, ta), __dmul_rn(2.0 * al * be, tc)), __dmul_rn(be * be, tb));
  double gs;                                                                // f = F + gs tau
  if (s.method == ANI_NEB_ASENEB) {
    const double mm = tt != 0.0 ? tt : 1.0;
    gs = climb ? -2.0 * ft / mm : -(ft + km * (al * ta + be * tc) - kp * (al * tc + be * tb)) / mm;
  } else if (tt > 0.0) {
    gs = climb ? -2.0 * ft / tt : -ft / tt + (kp * sqrt(tb) - km * sqrt(ta)) / sqrt(tt);
  } else {
    gs = 0.0;   // |tau| = 0: u = 0 (where ASE divides by zero)
  }
  g[0] = gs * al;
  g[1] = gs * be;
}

// launch 1: the block's partial sums {a, b, c, p, q} (grid: blocks per image x interior images)
__global__ void __launch_bounds__(NEB_BLOCK) k_neb_dots(const __grid_constant__ NebArgs a) {
  __shared__ double sv[ANI_NEB_DOTS * NEB_BLOCK], sw[NEB_BLOCK];
  const ani_neb_state& s = a.s;
  const int ci = blockIdx.y, j = blockIdx.x * NEB_BLOCK + threadIdx.x;
  if (a.step && ci == 0 && blockIdx.x == 0 && threadIdx.x == 0) s.fire.counter[1] = s.fire.counter[0];
  double d[ANI_NEB_DOTS] = {0.0, 0.0, 0.0, 0.0, 0.0}, w = 0.0;
  if (j < s.n_atoms) {
    double f[3], tm[3], tp[3];
    neb_vectors(a, ci, j, f, tm, tp);
    d[0] = tm[0] * tm[0] + tm[1] * tm[1] + tm[2] * tm[2];
    d[1] = tp[0] * tp[0] + tp[1] * tp[1] + tp[2] * tp[2];
    d[2] = tm[0] * tp[0] + tm[1] * tp[1] + tm[2] * tp[2];
    d[3] = f[0] * tm[0] + f[1] * tm[1] + f[2] * tm[2];
    d[4] = f[0] * tp[0] + f[1] * tp[1] + f[2] * tp[2];
  }
  block_reduce<ANI_NEB_DOTS>(d, w, sv, sw);
  if (threadIdx.x == 0) {
    double* out = s.dots + ANI_NEB_DOTS * ((size_t)ci * gridDim.x + blockIdx.x);
    for (int k = 0; k < ANI_NEB_DOTS; ++k) out[k] = d[k];
  }
}

// launch 2: the NEB forces of the block's atoms and their FIRE partials {f.v, f.f, v.v, max |f_i|^2}
__global__ void __launch_bounds__(NEB_BLOCK) k_neb_project(const __grid_constant__ NebArgs a) {
  __shared__ double sv[3 * NEB_BLOCK], sw[NEB_BLOCK], g[2];
  const ani_neb_state& s = a.s;
  const int ci = blockIdx.y, j = blockIdx.x * NEB_BLOCK + threadIdx.x, nb = gridDim.x;
  if (threadIdx.x == 0) {   // the image's partials, in block order
    double tot[ANI_NEB_DOTS] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int q = 0; q < nb; ++q) {
      const double* d = s.dots + ANI_NEB_DOTS * ((size_t)ci * nb + q);
      for (int k = 0; k < ANI_NEB_DOTS; ++k) tot[k] += d[k];
    }
    neb_gammas(a, ci, tot, g);
  }
  __syncthreads();
  double sum[3] = {0.0, 0.0, 0.0}, f2max = 0.0;
  if (j < s.n_atoms) {
    double f[3], tm[3], tp[3];
    neb_vectors(a, ci, j, f, tm, tp);
    const size_t k = (size_t)ci * s.n_atoms + j;
    const double* v = s.fire.v + 3 * k;
    double* out = s.neb_force + 3 * k;
    for (int d = 0; d < 3; ++d) {
      // 0 where force_scale is 0; the products rounded before the sum, so that a zero tangent adds exactly 0
      const double fd = f[d] + __dadd_rn(__dmul_rn(g[0], tm[d]), __dmul_rn(g[1], tp[d]));
      out[d] = fd;
      sum[0] += fd * v[d];
      sum[1] += fd * fd;
      sum[2] += v[d] * v[d];
    }
    f2max = sum[1];
  }
  block_reduce<3>(sum, f2max, sv, sw);
  if (threadIdx.x == 0) {
    double* p = s.fire.partials + 4 * ((size_t)ci * nb + blockIdx.x);
    p[0] = sum[0];
    p[1] = sum[1];
    p[2] = sum[2];
    p[3] = f2max;
  }
}

// launch 3: the band's totals, FIRE's scalars, the record, and the move to x(t+1)
__global__ void __launch_bounds__(NEB_BLOCK) k_neb_update(const __grid_constant__ NebArgs a) {
  __shared__ double cell[9], inv[9], mix[4];
  const ani_neb_state& s = a.s;
  const int m = s.n_images - 2, ci = blockIdx.y, b = ci / m, j = blockIdx.x * NEB_BLOCK + threadIdx.x;
  if (threadIdx.x < 32) {   // all of the band's partials, by fire_totals
    const int np = m * gridDim.x;
    double tot[4];
    fire_totals(s.fire.partials + 4 * (size_t)b * np, np, tot);
    if (threadIdx.x == 0) {
      const long long t = s.fire.counter[1];
      const bool leader = blockIdx.x == 0 && ci == b * m;
      const double* emax;
      const int imax = band_imax(a.energies, b, m, &emax);
      fire_scalars<ANI_NEB_RECORD>(s.fire, b, t, tot, leader, emax, mix);
      if (leader)
        s.fire.record[((size_t)(t % s.fire.record_rows) * s.fire.n_conf + b) * ANI_NEB_RECORD + 3] = (double)imax;
    }
  }
  load_cell(a.cells, a.cell_stride, ci, cell, inv);
  __syncthreads();
  if (mix[3] != 0.0 || j >= s.n_atoms) return;
  const size_t i = (size_t)ci * s.n_atoms + j;
  if (s.fire.force_scale[i] == 0.0) return;   // fixed and padding atoms: f = 0 and v = 0, so x never moves
  double xn[3];
  fire_move(mix, s.neb_force + 3 * i, s.fire.v + 3 * i, s.fire.x + 3 * i, xn);
  write_coords(a.coords, i, xn[0], xn[1], xn[2], a.cells, cell, inv);
}

// grid (blocks per image x interior images): with reset, v = 0 and the band's scalars of the current step; then the
// coordinates of x
__global__ void __launch_bounds__(NEB_BLOCK) k_neb_init(const __grid_constant__ NebArgs a) {
  __shared__ double cell[9], inv[9];
  const ani_neb_state& s = a.s;
  const int m = s.n_images - 2, ci = blockIdx.y, j = blockIdx.x * NEB_BLOCK + threadIdx.x;
  const size_t i = (size_t)ci * s.n_atoms + j;
  if (a.reset) {
    if (j < s.n_atoms)
      for (int d = 0; d < 3; ++d) s.fire.v[3 * i + d] = 0.0;
    if (ci % m == 0 && blockIdx.x == 0 && threadIdx.x == 0) fire_reset(s.fire, ci / m, s.fire.counter[0]);
  }
  load_cell(a.cells, a.cell_stride, ci, cell, inv);
  __syncthreads();
  if (j < s.n_atoms) write_coords(a.coords, i, s.fire.x[3 * i], s.fire.x[3 * i + 1], s.fire.x[3 * i + 2], a.cells, cell, inv);
}

bool neb_state_ok(const ani_neb_state* p) {
  if (!p) return false;
  const ani_opt_state& f = p->fire;
  return f.x && f.v && f.force_scale && f.params && f.scalars && f.counter && f.conv_step && f.record && f.partials &&
         f.record_rows >= 1 && p->endpoints && p->end_energies && p->springs && p->climb && p->neb_force && p->dots &&
         p->n_images >= 3 && p->n_atoms >= 1 && f.n_conf >= 1 &&
         (p->method == ANI_NEB_ASENEB || p->method == ANI_NEB_IMPROVED_TANGENT) &&
         (long long)f.n_per_conf == (long long)(p->n_images - 2) * p->n_atoms;
}

// the grid of every launch: (blocks per image, interior images); 0 when it does not fit
int neb_grid(const ani_neb_state* p, dim3* grid) {
  const long long imgs = (long long)p->fire.n_conf * (p->n_images - 2);
  const int rc = launch_shape(imgs, p->n_atoms);
  if (rc != ANI_OK) return rc;
  *grid = dim3((p->n_atoms + NEB_BLOCK - 1) / NEB_BLOCK, (unsigned)imgs);
  return ANI_OK;
}

int neb_launch(const ani_neb_state* state, const float* grad, const double* energies, const float* cells,
               int cell_stride, float* coords, bool step, void* stream) {
  if (!neb_state_ok(state) || !grad || !energies || (step && !coords)) return ANI_ERR_BAD_ARG;
  dim3 grid;
  const int rc = neb_grid(state, &grid);
  if (rc != ANI_OK) return rc;
  const NebArgs a = {{grad, energies, cells, cell_stride, coords, 0}, *state, step};
  cudaStream_t st = (cudaStream_t)stream;
  k_neb_dots<<<grid, NEB_BLOCK, 0, st>>>(a);
  k_neb_project<<<grid, NEB_BLOCK, 0, st>>>(a);
  if (step) k_neb_update<<<grid, NEB_BLOCK, 0, st>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

}  // namespace ani

using namespace ani;

extern "C" int ani_b200_neb_init(const ani_neb_state* state, const float* cells, int cell_mode, int reset,
                                 float* coords, void* stream) {
  NebArgs a = {};
  if (!neb_state_ok(state) || !coords || !init_cells(a, cells, cell_mode)) return ANI_ERR_BAD_ARG;
  dim3 grid;
  const int rc = neb_grid(state, &grid);
  if (rc != ANI_OK) return rc;
  a.s = *state;
  a.coords = coords;
  a.reset = reset != 0;
  k_neb_init<<<grid, NEB_BLOCK, 0, (cudaStream_t)stream>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_neb_step(const ani_neb_state* state, const float* grad, const double* energies,
                                 const float* cell, float* coords, void* stream) {
  return neb_launch(state, grad, energies, cell, 0, coords, true, stream);
}

extern "C" int ani_b200_neb_step_cells(const ani_neb_state* state, const float* grad, const double* energies,
                                       const float* lattice, float* coords, void* stream) {
  if (!lattice) return ANI_ERR_BAD_ARG;
  return neb_launch(state, grad, energies, lattice, ANI_LATTICE_STRIDE, coords, true, stream);
}

extern "C" int ani_b200_neb_project(const ani_neb_state* state, const float* grad, const double* energies,
                                    void* stream) {
  return neb_launch(state, grad, energies, nullptr, 0, nullptr, false, stream);
}
