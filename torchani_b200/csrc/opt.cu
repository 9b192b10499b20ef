// Geometry optimisation on the device: FIRE, as ASE's ase.optimize.FIRE defines it (without its downhill check), one
// independent optimisation per conformer.  The master positions and FIRE velocities (float64) and the per-conformer
// scalars {dt, a, n} stay in device memory and the launches write the float32 coordinates of the next force step, so
// K whole steps (FIRE + force step) capture into one CUDA graph, as the MD steps of md.cu do.
//
// One step is the force step at x(t) followed by two launches of this file (ani_b200_opt_step):
//   k_opt_reduce  per block of ANI_MD_BLOCK atoms of a conformer: the partial sums P = f.v, F2 = f.f, V2 = v.v and the
//                 largest |f_i|^2, with f = -dE/dx * force_scale (eV / A; 0 for fixed and padding atoms)
//   k_opt_update  per block: the conformer's partials summed in a fixed order (every block of the conformer forms the
//                 same totals, and from them the same mixing coefficients and step scale); block 0 writes the record
//                 of step t, the convergence step and the scalars of step t + 1; then v' and x(t+1) of the block's
//                 atoms, and the float32 coordinates of x(t+1), wrapped into the cell
// The norm of the step comes from the same three sums as the mixing, |dr|^2 = dt^2 |c1 v + (c2 + dt) f|^2, so no second
// reduction runs after v'.  The scalars are double-buffered by step parity (step t reads slot t % 2, block 0 writes
// slot (t + 1) % 2): no launch reads a word another block of the same launch writes.  Every sum is float64 in a fixed
// order (block trees of fixed shape, no atomics): two runs from the same state and forces give identical bits.  The
// step counter lives on the device with the protocol of md.cu.
//
// Variable cell (ani_b200_opt_cell_step, the CELL instances of the same two launches): FIRE on the degrees of freedom
// of ASE's FrechetCellFilter, A atom rows u = F^-1 r (s.x holds u) and 3 cell rows d = c logm(F), with the cell
// h = h0 F^T.  k_opt_reduce transforms every atom row by F(t)^T, and its block 0 also sums the conformer's virial slots
// (in a fixed order), forms the cell force Phi, writes it to cell_force and adds the cell rows to its partials.
// k_opt_update moves the cell rows with the atom rows, and every block forms F(t+1) = expm(d(t+1) / c) by the same code
// from the same inputs (so the same bits) to write the float32 coordinates F(t+1) u(t+1), wrapped into the
// float32-rounded h0 F(t+1)^T.  The master {d, v_cell, F} is double-buffered by step parity like the scalars: block 0
// writes slot (t + 1) % 2 and the float32 cell of the next force step, which no block of the step reads.
#include "md_common.cuh"

namespace ani {

constexpr int OPT_BLOCK = ANI_MD_BLOCK;

struct OptArgs : LoopArgs {
  ani_opt_state s;
};

struct OptCellArgs : OptArgs {
  ani_opt_cell q;
};

template <bool CELL>
struct OptArgsOf {
  using type = OptArgs;
};
template <>
struct OptArgsOf<true> {
  using type = OptCellArgs;
};

// c = a b (3 x 3, row-major)
__device__ __forceinline__ void mm3(const double* a, const double* b, double* c) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) c[3 * i + j] = a[3 * i] * b[j] + a[3 * i + 1] * b[3 + j] + a[3 * i + 2] * b[6 + j];
}

constexpr int EXPM_TERMS = 13;   // |A / 2^s|_1 <= 1/4: the first term left out is < 0.25^14 / 14! < 1e-20

// x = expm(a) and, with FRECHET, q = D_expm(a)[e], the Frechet derivative in the direction e (3 x 3, float64): the
// Taylor series of the block matrix [[a, e], [0, a]] / 2^s by Horner's rule, then s squarings.  Its products keep the
// block form [[x, q], [0, x]], so each costs three 3 x 3 products; the error of q is relative to |e| (q is linear in e).
template <bool FRECHET>
__device__ __noinline__ void expm3(const double* a, const double* e, double* x, double* q) {
  double nrm = 0.0;
  for (int j = 0; j < 3; ++j) nrm = fmax(nrm, fabs(a[j]) + fabs(a[3 + j]) + fabs(a[6 + j]));
  int s = 0;
  if (nrm > 0.25) {
    frexp(4.0 * nrm, &s);   // 4 nrm < 2^s
    s = min(max(s, 0), 1100);
  }
  const double sc = ldexp(1.0, -s);
  double as[9], es[9], t[9], u[9];
  for (int k = 0; k < 9; ++k) {
    as[k] = a[k] * sc;
    if (FRECHET) es[k] = e[k] * sc;
    x[k] = (k % 4 == 0) ? 1.0 : 0.0;
    if (FRECHET) q[k] = 0.0;
  }
#pragma unroll 1
  for (int n = EXPM_TERMS; n >= 1; --n) {   // [x, q] <- I + [[as, es], [0, as]] [x, q] / n
    const double r = 1.0 / n;
    mm3(as, x, t);
    if (FRECHET) {
      mm3(as, q, u);
      mm3(es, x, q);
      for (int k = 0; k < 9; ++k) q[k] = (u[k] + q[k]) * r;
    }
    for (int k = 0; k < 9; ++k) x[k] = t[k] * r + ((k % 4 == 0) ? 1.0 : 0.0);
  }
#pragma unroll 1
  for (int k = 0; k < s; ++k) {   // [x, q]^2 = [x x, x q + q x]
    if (FRECHET) {
      mm3(x, q, t);
      mm3(q, x, u);
      for (int m = 0; m < 9; ++m) q[m] = t[m] + u[m];
    }
    mm3(x, x, t);
    for (int m = 0; m < 9; ++m) x[m] = t[m];
  }
}

// the master {d, v_cell, F} of conformer c at step t
__device__ __forceinline__ double* cell_slot(const ani_opt_cell& q, int n_conf, int c, long long t) {
  return q.master + ((size_t)(t & 1) * n_conf + c) * ANI_OPT_CELL_MASTER;
}

// h = h0 F^T
__device__ __forceinline__ void deformed_cell(const double* h0, const double* f, double* h) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) h[3 * i + j] = h0[3 * i] * f[3 * j] + h0[3 * i + 1] * f[3 * j + 1] + h0[3 * i + 2] * f[3 * j + 2];
}

// the cell rows of conformer c at step t, by warp 0 of the conformer's block 0 (k_opt_reduce): the virial slots summed
// lane-strided in order and then by a fixed tree towards lane 0, which forms Phi, writes it to cell_force and the record
// {V, -tr W / (3 V), E + p0 V} of step t, and returns the cell rows' {P, F2, V2, max row^2} in part
__device__ void cell_rows(const OptCellArgs& a, int c, long long t, double* part) {
  const ani_opt_cell& q = a.q;
  const double* vs = q.virial + (size_t)c * q.virial_slots * 9;
  double w[9];
  warp_reduce<9, 0>(threadIdx.x, q.virial_slots, [&](int b, double* v) {
    for (int k = 0; k < 9; ++k) v[k] = vs[9 * b + k];
  }, w);
  if (threadIdx.x != 0) return;
  const double* m = cell_slot(q, a.s.n_conf, c, t);
  const double *d = m, *vc = m + 9, *f = m + 18;
  const double* par = q.params + (size_t)c * ANI_OPT_CELL_PARAMS;   // p0, c, unit
  double h[9], fi[9], g[9], lt[9], phi[9];
  deformed_cell(q.h0 + (size_t)c * 9, f, h);
  const double vol = fabs(det3(h));
  invert3(f, fi);
  // G = -(W + p0 V I) F^-T unit
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double acc = 0.0;
      for (int k = 0; k < 3; ++k) acc += (w[3 * i + k] + (i == k ? par[0] * vol : 0.0)) * fi[3 * j + k];
      g[3 * i + j] = -acc * par[2];
    }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) lt[3 * i + j] = d[3 * j + i] / par[1];
  expm3<true>(lt, g, h, phi);   // (h: the exponential, unused)
  const double tr3 = (phi[0] + phi[4] + phi[8]) / (3.0 * par[1]);
  for (int k = 0; k < 9; ++k) {
    phi[k] /= par[1];
    if (q.projection == 1) phi[k] = (k % 4 == 0) ? tr3 : 0.0;
    else if (q.projection == 2 && k % 4 == 0) phi[k] -= tr3;
  }
  double* out = q.cell_force + (size_t)c * 9;
  part[0] = part[1] = part[2] = part[3] = 0.0;
  for (int r = 0; r < 3; ++r) {
    double rr = 0.0;
    for (int k = 3 * r; k < 3 * r + 3; ++k) {
      out[k] = phi[k];
      part[0] += phi[k] * vc[k];
      rr += phi[k] * phi[k];
      part[2] += vc[k] * vc[k];
    }
    part[1] += rr;
    part[3] = fmax(part[3], rr);
  }
  double* rec = q.record + ((size_t)(t % a.s.record_rows) * a.s.n_conf + c) * ANI_OPT_CELL_RECORD;
  rec[0] = vol;
  rec[1] = -(w[0] + w[4] + w[8]) / (3.0 * vol);
  rec[2] = a.energies[c] + par[0] * vol;
}

// launch 1 of a step: the per-block partials {P, F2, V2, max |f_i|^2} (grid: blocks per conformer x conformers); with
// CELL the atom rows are f F(t) and block 0 adds the cell rows
template <bool CELL>
__global__ void __launch_bounds__(OPT_BLOCK) k_opt_reduce(const __grid_constant__ typename OptArgsOf<CELL>::type a) {
  __shared__ double sv[3 * OPT_BLOCK], sw[OPT_BLOCK];
  const ani_opt_state& s = a.s;
  const int c = blockIdx.y, j = blockIdx.x * OPT_BLOCK + threadIdx.x;
  if (c == 0 && blockIdx.x == 0 && threadIdx.x == 0) s.counter[1] = s.counter[0];
  double sum[3] = {0.0, 0.0, 0.0}, f2max = 0.0;
  if (j < s.n_per_conf) {
    const size_t i = (size_t)c * s.n_per_conf + j;
    const double fs = s.force_scale[i];
    double fx = -(double)a.grad[3 * i + 0] * fs, fy = -(double)a.grad[3 * i + 1] * fs,
           fz = -(double)a.grad[3 * i + 2] * fs;
    if constexpr (CELL) {   // g = f F(t) (counter[0]: written by the previous launch only)
      const double* f = cell_slot(a.q, s.n_conf, c, s.counter[0]) + 18;
      const double gx = fx * f[0] + fy * f[3] + fz * f[6], gy = fx * f[1] + fy * f[4] + fz * f[7];
      fz = fx * f[2] + fy * f[5] + fz * f[8];
      fx = gx;
      fy = gy;
    }
    const double vx = s.v[3 * i + 0], vy = s.v[3 * i + 1], vz = s.v[3 * i + 2];
    sum[0] = fx * vx + fy * vy + fz * vz;
    sum[1] = fx * fx + fy * fy + fz * fz;
    sum[2] = vx * vx + vy * vy + vz * vz;
    f2max = sum[1];
  }
  [[maybe_unused]] double cp[4];
  if constexpr (CELL) {
    if (blockIdx.x == 0 && threadIdx.x < 32) cell_rows(a, c, s.counter[0], cp);
  }
  block_reduce<3>(sum, f2max, sv, sw);
  if (threadIdx.x == 0) {
    if constexpr (CELL) {
      if (blockIdx.x == 0) {   // the cell rows after the atom rows' tree
        sum[0] += cp[0];
        sum[1] += cp[1];
        sum[2] += cp[2];
        f2max = fmax(f2max, cp[3]);
      }
    }
    double* p = s.partials + 4 * ((size_t)c * gridDim.x + blockIdx.x);
    p[0] = sum[0];
    p[1] = sum[1];
    p[2] = sum[2];
    p[3] = f2max;
  }
}

// the cell rows' move of conformer c at step t by thread 0 of every block (k_opt_update), after fire_scalars: from
// slot t % 2 and cell_force, v_cell' = c1 v_cell + (c2 + dt) Phi, d(t+1) = d + s v_cell' and F(t+1) = expm(d(t+1) / c)
// (all unchanged for a frozen conformer); F(t) to cell[9..18), F(t+1) to cell[18..27), the float32-rounded
// h0 F(t+1)^T to cell[0..9) and its inverse to inv.  Block 0 writes slot (t + 1) % 2 and the float32 cell.
__device__ void cell_move(const OptCellArgs& a, int c, long long t, const double* mix, double* cell, double* inv) {
  const ani_opt_cell& q = a.q;
  const double* m = cell_slot(q, a.s.n_conf, c, t);
  const double* phi = q.cell_force + (size_t)c * 9;
  const double* par = q.params + (size_t)c * ANI_OPT_CELL_PARAMS;
  double dn[18], h[9];   // d(t+1), v_cell'
  for (int k = 0; k < 9; ++k) {
    cell[9 + k] = m[18 + k];
    dn[9 + k] = mix[3] != 0.0 ? m[9 + k] : mix[0] * m[9 + k] + mix[1] * phi[k];
    dn[k] = mix[3] != 0.0 ? m[k] : m[k] + mix[2] * dn[9 + k];
  }
  double* fn = cell + 18;
  if (mix[3] != 0.0) {
    for (int k = 0; k < 9; ++k) fn[k] = m[18 + k];
  } else {
    double ln[9];
    for (int k = 0; k < 9; ++k) ln[k] = dn[k] / par[1];
    expm3<false>(ln, nullptr, fn, nullptr);
  }
  deformed_cell(q.h0 + (size_t)c * 9, fn, h);
  for (int k = 0; k < 9; ++k) cell[k] = (double)(float)h[k];
  invert3(cell, inv);
  if (blockIdx.x != 0) return;
  double* mn = cell_slot(q, a.s.n_conf, c, t + 1);
  float* out = q.cell_out + (size_t)c * q.cell_stride;
  for (int k = 0; k < 9; ++k) {
    mn[k] = dn[k];
    mn[9 + k] = dn[9 + k];
    mn[18 + k] = fn[k];
    out[k] = (float)h[k];
  }
}

// launch 2 of a step: totals, record, convergence check, scalars, and the move to x(t+1) (with CELL: to u(t+1), d(t+1))
template <bool CELL>
__global__ void __launch_bounds__(OPT_BLOCK) k_opt_update(const __grid_constant__ typename OptArgsOf<CELL>::type a) {
  __shared__ double cell[CELL ? 27 : 9], inv[9], mix[4];   // CELL: then F(t), F(t+1)
  const ani_opt_state& s = a.s;
  const int c = blockIdx.y, j = blockIdx.x * OPT_BLOCK + threadIdx.x, nb = gridDim.x;
  if (threadIdx.x < 32) {   // the conformer's partials, by fire_totals
    double tot[4];
    fire_totals(s.partials + 4 * (size_t)c * nb, nb, tot);
    if (threadIdx.x == 0) {
      fire_scalars<ANI_OPT_RECORD>(s, c, s.counter[1], tot, blockIdx.x == 0, a.energies + c, mix);
      if constexpr (CELL) cell_move(a, c, s.counter[1], mix, cell, inv);
    }
  }
  if constexpr (!CELL) load_cell(a.cells, a.cell_stride, c, cell, inv);
  __syncthreads();
  if (mix[3] != 0.0 || j >= s.n_per_conf) return;
  const size_t i = (size_t)c * s.n_per_conf + j;
  const double fs = s.force_scale[i];
  if (fs == 0.0) return;   // fixed and padding atoms: f = 0 and v = 0, so x never moves
  double fx = -(double)a.grad[3 * i + 0] * fs, fy = -(double)a.grad[3 * i + 1] * fs,
         fz = -(double)a.grad[3 * i + 2] * fs;
  if constexpr (CELL) {   // g = f F(t), as in k_opt_reduce
    const double* f = cell + 9;
    const double gx = fx * f[0] + fy * f[3] + fz * f[6], gy = fx * f[1] + fy * f[4] + fz * f[7];
    fz = fx * f[2] + fy * f[5] + fz * f[8];
    fx = gx;
    fy = gy;
  }
  const double f[3] = {fx, fy, fz};
  double xn[3];
  fire_move(mix, f, s.v + 3 * i, s.x + 3 * i, xn);
  const double x = xn[0], y = xn[1], z = xn[2];
  if constexpr (CELL) {   // r = F(t+1) u(t+1), wrapped into the float32-rounded h0 F(t+1)^T
    const double* f = cell + 18;
    write_coords(a.coords, i, f[0] * x + f[1] * y + f[2] * z, f[3] * x + f[4] * y + f[5] * z,
                 f[6] * x + f[7] * y + f[8] * z, true, cell, inv);
  } else {
    write_coords(a.coords, i, x, y, z, a.cells, cell, inv);
  }
}

// one CTA per conformer: with reset, v = 0 and the scalars of the current step; then the coordinates of x
__global__ void __launch_bounds__(OPT_BLOCK) k_opt_init(const __grid_constant__ OptArgs a) {
  const ani_opt_state& s = a.s;
  const int c = blockIdx.x, A = s.n_per_conf;
  if (a.reset) {
    for (int j = threadIdx.x; j < 3 * A; j += OPT_BLOCK) s.v[3 * (size_t)c * A + j] = 0.0;
    if (threadIdx.x == 0) fire_reset(s, c, s.counter[0]);
  }
  conformer_coords(a, c, A, s.x);
}

// one CTA per conformer: with reset, v = 0, the scalars of the current step and the master {0, 0, I}; then the float32
// cell h0 F^T and the coordinates of F u wrapped into it
__global__ void __launch_bounds__(OPT_BLOCK) k_opt_cell_init(const __grid_constant__ OptCellArgs a) {
  __shared__ double cell[9], inv[9], f[9];
  const ani_opt_state& s = a.s;
  const ani_opt_cell& q = a.q;
  const int c = blockIdx.x, A = s.n_per_conf;
  const size_t base = (size_t)c * A;
  const long long t = s.counter[0];
  double* m = cell_slot(q, s.n_conf, c, t);
  if (a.reset) {
    for (int j = threadIdx.x; j < 3 * A; j += OPT_BLOCK) s.v[3 * base + j] = 0.0;
    if (threadIdx.x == 0) {
      fire_reset(s, c, t);
      for (int k = 0; k < 18; ++k) m[k] = 0.0;
      for (int k = 0; k < 9; ++k) m[18 + k] = (k % 4 == 0) ? 1.0 : 0.0;
    }
  }
  if (threadIdx.x == 0) {
    double h[9];
    for (int k = 0; k < 9; ++k) f[k] = m[18 + k];
    deformed_cell(q.h0 + (size_t)c * 9, f, h);
    float* out = q.cell_out + (size_t)c * q.cell_stride;
    for (int k = 0; k < 9; ++k) {
      cell[k] = (double)(float)h[k];
      out[k] = (float)h[k];
    }
    invert3(cell, inv);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < A; j += OPT_BLOCK) {
    const size_t i = base + j;
    const double x = s.x[3 * i + 0], y = s.x[3 * i + 1], z = s.x[3 * i + 2];
    write_coords(a.coords, i, f[0] * x + f[1] * y + f[2] * z, f[3] * x + f[4] * y + f[5] * z,
                 f[6] * x + f[7] * y + f[8] * z, true, cell, inv);
  }
}

bool opt_state_ok(const ani_opt_state* s) {
  return s && s->x && s->v && s->force_scale && s->params && s->scalars && s->counter && s->n_conf >= 1 &&
         s->n_per_conf >= 1;
}

int opt_step(const ani_opt_state* s, const float* grad, const double* energies, const float* cells, int cell_stride,
             float* coords, void* stream) {
  if (!opt_state_ok(s) || !s->conv_step || !s->record || !s->partials || s->record_rows < 1) return ANI_ERR_BAD_ARG;
  if (!grad || !energies || !coords) return ANI_ERR_BAD_ARG;
  const int rc = launch_shape(s->n_conf, s->n_per_conf);
  if (rc != ANI_OK) return rc;
  const OptArgs a = {{grad, energies, cells, cell_stride, coords, 0}, *s};
  const dim3 grid((s->n_per_conf + OPT_BLOCK - 1) / OPT_BLOCK, s->n_conf);
  cudaStream_t st = (cudaStream_t)stream;
  k_opt_reduce<false><<<grid, OPT_BLOCK, 0, st>>>(a);
  k_opt_update<false><<<grid, OPT_BLOCK, 0, st>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

bool opt_cell_ok(const ani_opt_cell* q) {
  return q && q->master && q->h0 && q->params && q->cell_out && q->virial && q->cell_force && q->record &&
         q->cell_stride >= 9 && q->virial_slots >= 1 && q->projection >= 0 && q->projection <= 2;
}

}  // namespace ani

using namespace ani;

extern "C" int ani_b200_opt_init(const ani_opt_state* state, const float* cells, int cell_mode, int reset,
                                 float* coords, void* stream) {
  OptArgs a = {};
  if (!opt_state_ok(state) || !coords || !init_cells(a, cells, cell_mode)) return ANI_ERR_BAD_ARG;
  a.s = *state;
  a.coords = coords;
  a.reset = reset != 0;
  k_opt_init<<<state->n_conf, OPT_BLOCK, 0, (cudaStream_t)stream>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_opt_step(const ani_opt_state* state, const float* grad, const double* energies,
                                 const float* cell, float* coords, void* stream) {
  return opt_step(state, grad, energies, cell, 0, coords, stream);
}

extern "C" int ani_b200_opt_step_cells(const ani_opt_state* state, const float* grad, const double* energies,
                                       const float* lattice, float* coords, void* stream) {
  if (!lattice) return ANI_ERR_BAD_ARG;
  return opt_step(state, grad, energies, lattice, ANI_LATTICE_STRIDE, coords, stream);
}

extern "C" int ani_b200_opt_cell_init(const ani_opt_state* state, const ani_opt_cell* cell, int reset, float* coords,
                                      void* stream) {
  if (!opt_state_ok(state) || !opt_cell_ok(cell) || !coords) return ANI_ERR_BAD_ARG;
  OptCellArgs a = {};
  a.s = *state;
  a.q = *cell;
  a.coords = coords;
  a.reset = reset != 0;
  k_opt_cell_init<<<state->n_conf, OPT_BLOCK, 0, (cudaStream_t)stream>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_opt_cell_step(const ani_opt_state* state, const ani_opt_cell* cell, const float* grad,
                                      const double* energies, float* coords, void* stream) {
  const ani_opt_state* s = state;
  if (!opt_state_ok(s) || !s->conv_step || !s->record || !s->partials || s->record_rows < 1) return ANI_ERR_BAD_ARG;
  if (!opt_cell_ok(cell) || !grad || !energies || !coords) return ANI_ERR_BAD_ARG;
  const int rc = launch_shape(s->n_conf, s->n_per_conf);
  if (rc != ANI_OK) return rc;
  const OptCellArgs a = {{{grad, energies, nullptr, 0, coords, 0}, *s}, *cell};
  const dim3 grid((s->n_per_conf + OPT_BLOCK - 1) / OPT_BLOCK, s->n_conf);
  cudaStream_t st = (cudaStream_t)stream;
  k_opt_reduce<true><<<grid, OPT_BLOCK, 0, st>>>(a);
  k_opt_update<true><<<grid, OPT_BLOCK, 0, st>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}
