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
#include "md_common.cuh"

namespace ani {

constexpr int OPT_BLOCK = ANI_MD_BLOCK;

struct OptArgs {
  ani_opt_state s;
  const float* grad;          // f32[n][3] dE/dx (Hartree / A), input order
  const double* energies;     // f64[n_conf]
  const float* cells;         // cell rows (f32[9]) of conformer c at cells + c * cell_stride; nullptr = open
  int cell_stride;
  float* coords;              // f32[n][3]
  int reset;                  // (ani_b200_opt_init)
};

// launch 1 of a step: the per-block partials {P, F2, V2, max |f_i|^2} (grid: blocks per conformer x conformers)
__global__ void __launch_bounds__(OPT_BLOCK) k_opt_reduce(const __grid_constant__ OptArgs a) {
  __shared__ double sv[3 * OPT_BLOCK], sw[OPT_BLOCK];
  const ani_opt_state& s = a.s;
  const int c = blockIdx.y, j = blockIdx.x * OPT_BLOCK + threadIdx.x;
  if (c == 0 && blockIdx.x == 0 && threadIdx.x == 0) s.counter[1] = s.counter[0];
  double sum[3] = {0.0, 0.0, 0.0}, f2max = 0.0;
  if (j < s.n_per_conf) {
    const size_t i = (size_t)c * s.n_per_conf + j;
    const double fs = s.force_scale[i];
    const double fx = -(double)a.grad[3 * i + 0] * fs, fy = -(double)a.grad[3 * i + 1] * fs,
                 fz = -(double)a.grad[3 * i + 2] * fs;
    const double vx = s.v[3 * i + 0], vy = s.v[3 * i + 1], vz = s.v[3 * i + 2];
    sum[0] = fx * vx + fy * vy + fz * vz;
    sum[1] = fx * fx + fy * fy + fz * fz;
    sum[2] = vx * vx + vy * vy + vz * vz;
    f2max = sum[1];
  }
  block_reduce<3>(sum, f2max, sv, sw);
  if (threadIdx.x == 0) {
    double* p = s.partials + 4 * ((size_t)c * gridDim.x + blockIdx.x);
    p[0] = sum[0];
    p[1] = sum[1];
    p[2] = sum[2];
    p[3] = f2max;
  }
}

// FIRE's scalar update of conformer c at step t from the totals {P, F2, V2, max |f_i|^2}, by thread 0 of every block
// of the conformer (the same inputs, so the same results everywhere): mix = {c1, c2 + dt, dt * min(1, maxstep / |dr|),
// frozen}.  Block 0 writes the record of step t, the convergence step and the scalars of step t + 1.
__device__ void fire_scalars(const OptArgs& a, int c, long long t, const double* tot, double* mix) {
  const ani_opt_state& s = a.s;
  const double* par = s.params + (size_t)c * ANI_OPT_PARAMS;   // dt0, maxstep, dtmax, Nmin, finc, fdec, astart, fa, fmax
  const double* sc = s.scalars + ((size_t)(t & 1) * s.n_conf + c) * ANI_OPT_SCALARS;
  const double p = tot[0], f2 = tot[1], v2 = tot[2], fmax_ = sqrt(tot[3]);
  double dt = sc[0], al = sc[1], n = sc[2];
  // conv_step[c] is written below by block 0 of this conformer only, and only with the value t: a block that reads it
  // concurrently sees -1 or t, and "converged before this step" is false for both
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
  if (blockIdx.x != 0) return;
  double* nx = s.scalars + ((size_t)((t + 1) & 1) * s.n_conf + c) * ANI_OPT_SCALARS;
  nx[0] = dt;
  nx[1] = al;
  nx[2] = n;
  double* row = s.record + ((size_t)(t % s.record_rows) * s.n_conf + c) * ANI_OPT_RECORD;
  row[0] = (double)t;
  row[1] = a.energies[c];
  row[2] = fmax_;
  if (conv) s.conv_step[c] = t;
  if (c == 0) s.counter[0] = t + 1;
}

// launch 2 of a step: totals, record, convergence check, scalars, and the move to x(t+1)
__global__ void __launch_bounds__(OPT_BLOCK) k_opt_update(const __grid_constant__ OptArgs a) {
  __shared__ double cell[9], inv[9], mix[4];
  const ani_opt_state& s = a.s;
  const int c = blockIdx.y, j = blockIdx.x * OPT_BLOCK + threadIdx.x, nb = gridDim.x;
  if (threadIdx.x < 32) {   // the conformer's partials: lane-strided in order, then a fixed tree towards lane 0
    double tot[4] = {0.0, 0.0, 0.0, 0.0};
    for (int b = threadIdx.x; b < nb; b += 32) {
      const double* q = s.partials + 4 * ((size_t)c * nb + b);
      tot[0] += q[0];
      tot[1] += q[1];
      tot[2] += q[2];
      tot[3] = fmax(tot[3], q[3]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      tot[0] += __shfl_down_sync(ANI_FULL_MASK, tot[0], o);
      tot[1] += __shfl_down_sync(ANI_FULL_MASK, tot[1], o);
      tot[2] += __shfl_down_sync(ANI_FULL_MASK, tot[2], o);
      tot[3] = fmax(tot[3], __shfl_down_sync(ANI_FULL_MASK, tot[3], o));
    }
    if (threadIdx.x == 0) fire_scalars(a, c, s.counter[1], tot, mix);
  }
  load_cell(a.cells, a.cell_stride, c, cell, inv);
  __syncthreads();
  if (mix[3] != 0.0 || j >= s.n_per_conf) return;
  const size_t i = (size_t)c * s.n_per_conf + j;
  const double fs = s.force_scale[i];
  if (fs == 0.0) return;   // fixed and padding atoms: f = 0 and v = 0, so x never moves
  const double c1 = mix[0], cf = mix[1], st = mix[2];
  const double vx = c1 * s.v[3 * i + 0] + cf * (-(double)a.grad[3 * i + 0] * fs);
  const double vy = c1 * s.v[3 * i + 1] + cf * (-(double)a.grad[3 * i + 1] * fs);
  const double vz = c1 * s.v[3 * i + 2] + cf * (-(double)a.grad[3 * i + 2] * fs);
  const double x = s.x[3 * i + 0] + st * vx, y = s.x[3 * i + 1] + st * vy, z = s.x[3 * i + 2] + st * vz;
  s.v[3 * i + 0] = vx;
  s.v[3 * i + 1] = vy;
  s.v[3 * i + 2] = vz;
  s.x[3 * i + 0] = x;
  s.x[3 * i + 1] = y;
  s.x[3 * i + 2] = z;
  write_coords(a.coords, i, x, y, z, a.cells, cell, inv);
}

// one CTA per conformer: with reset, v = 0 and the scalars of the current step; then the coordinates of x
__global__ void __launch_bounds__(OPT_BLOCK) k_opt_init(const __grid_constant__ OptArgs a) {
  __shared__ double cell[9], inv[9];
  const ani_opt_state& s = a.s;
  const int c = blockIdx.x, A = s.n_per_conf;
  const size_t base = (size_t)c * A;
  if (a.reset) {
    for (int j = threadIdx.x; j < 3 * A; j += OPT_BLOCK) s.v[3 * base + j] = 0.0;
    if (threadIdx.x == 0) {
      const double* par = s.params + (size_t)c * ANI_OPT_PARAMS;
      double* sc = s.scalars + ((size_t)(s.counter[0] & 1) * s.n_conf + c) * ANI_OPT_SCALARS;
      sc[0] = par[0];
      sc[1] = par[6];
      sc[2] = 0.0;
    }
  }
  load_cell(a.cells, a.cell_stride, c, cell, inv);
  __syncthreads();
  for (int j = threadIdx.x; j < A; j += OPT_BLOCK) {
    const size_t i = base + j;
    write_coords(a.coords, i, s.x[3 * i + 0], s.x[3 * i + 1], s.x[3 * i + 2], a.cells, cell, inv);
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
  if ((long long)s->n_conf * s->n_per_conf > 0x7fffffffLL || s->n_conf > 65535) return ANI_ERR_UNSUPPORTED;
  OptArgs a = {};
  a.s = *s;
  a.grad = grad;
  a.energies = energies;
  a.cells = cells;
  a.cell_stride = cell_stride;
  a.coords = coords;
  const dim3 grid((s->n_per_conf + OPT_BLOCK - 1) / OPT_BLOCK, s->n_conf);
  cudaStream_t st = (cudaStream_t)stream;
  k_opt_reduce<<<grid, OPT_BLOCK, 0, st>>>(a);
  k_opt_update<<<grid, OPT_BLOCK, 0, st>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

}  // namespace ani

using namespace ani;

extern "C" int ani_b200_opt_init(const ani_opt_state* state, const float* cells, int cell_mode, int reset,
                                 float* coords, void* stream) {
  if (!opt_state_ok(state) || !coords || cell_mode < 0 || cell_mode > 2 || (cell_mode && !cells))
    return ANI_ERR_BAD_ARG;
  OptArgs a = {};
  a.s = *state;
  a.cells = cell_mode ? cells : nullptr;
  a.cell_stride = cell_mode == 2 ? 9 : 0;
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
