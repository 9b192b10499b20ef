// Molecular dynamics on the device: velocity Verlet and BAOAB Langevin integrators that keep the master positions and
// velocities (float64) in device memory and write the float32 coordinates of the next force step, so that K whole MD
// steps (integrator + force step) capture into one CUDA graph.
//
// One MD step is the force step at x(t) followed by two launches of this file (ani_b200_md_step):
//   k_md_finish   per atom: the final half kick B(dt/2) with the forces at x(t), giving v(t) (not at t = 0, where v(0)
//                 is the initial velocity); per block of ANI_MD_BLOCK atoms of a conformer: the partial kinetic energy
//                 and the largest force_relative_stdev
//   k_md_start    per block: the conformer's partials summed in a fixed order (every block of the conformer forms the
//                 same totals); block 0 writes the thermo record of step t; the frame of step t; the stop check; then
//                 B(dt/2) A(dt) (velocity Verlet) or B(dt/2) A(dt/2) O(dt) A(dt/2) (BAOAB) and the float32
//                 coordinates of x(t+1), wrapped into the cell
// Every sum is float64 in a fixed order (block trees of fixed shape, no atomics): two runs from the same state and
// forces give identical bits.  The step counter lives on the device (counter[0] is read by k_md_finish, which copies
// it to counter[1] for k_md_start, which advances counter[0]), so a replayed graph needs no argument changes.
//
// Constant pressure (ani_b200_md_step_npt): k_md_start also forms the conformer's internal pressure from E_kin, the
// trace of the force step's virial and the volume of its float64 master cell, draws the isotropic stochastic cell
// rescaling (Bernetti & Bussi 2020) factor mu, and after B A (O A) scales x and the cell by mu and v by 1 / mu.  The
// master cell is double-buffered by step parity (step t reads slot t % 2, block 0 writes slot (t + 1) % 2), and the
// float32 coordinates are wrapped into the float32-rounded new cell, which block 0 also writes for the next force
// step's preparation: no launch reads a word another block of the same launch writes.
#include "md_common.cuh"

namespace ani {

constexpr int MD_BLOCK = ANI_MD_BLOCK;

struct MdArgs : LoopArgs {
  ani_md_state s;
  const double* qbc;          // f64[n_conf] or nullptr (no stop check)
  const float* force_stdev;   // f32[n] force_relative_stdev or nullptr
  ani_md_barostat baro;       // ani_b200_md_step_npt; baro.master == nullptr for NVE / NVT
};

// ---- counter-based normals: Philox4x32-10 keyed on the seed, counter (step, atom, component) ----------------------
__host__ __device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
    const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    c[0] = hi1 ^ c[1] ^ k0;
    c[1] = lo1;
    c[2] = hi0 ^ c[3] ^ k1;
    c[3] = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}

// (a, b) -> a uniform double in (0, 1) from their top 53 bits
__device__ __forceinline__ double unit_open(uint32_t a, uint32_t b) {
  const uint64_t m = (((uint64_t)a << 32) | b) >> 11;
  return ((double)m + 0.5) * 0x1.0p-53;
}

// standard normal of (seed, step, atom, component): one Philox block, Box-Muller (cosine branch)
__device__ __forceinline__ double md_normal(unsigned long long seed, long long step, int atom, int comp) {
  uint32_t c[4] = {(uint32_t)(unsigned long long)step, (uint32_t)((unsigned long long)step >> 32), (uint32_t)atom,
                   (uint32_t)comp};
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  const double u1 = unit_open(c[0], c[1]), u2 = unit_open(c[2], c[3]);
  return sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
}

// launch 1 of a step: the final half kick and the per-block partial sums (grid: blocks per conformer x conformers)
__global__ void __launch_bounds__(MD_BLOCK) k_md_finish(const __grid_constant__ MdArgs a) {
  __shared__ double sv[MD_BLOCK], sw[MD_BLOCK];
  const ani_md_state& s = a.s;
  const int c = blockIdx.y, j = blockIdx.x * MD_BLOCK + threadIdx.x;
  const long long t = s.counter[0];
  if (c == 0 && blockIdx.x == 0 && threadIdx.x == 0) s.counter[1] = t;
  const bool frozen = s.stop_step[c] >= 0;
  const double dt = s.params[(size_t)c * ANI_MD_PARAMS + 0];
  double ke = 0.0, fmax_ = 0.0;
  if (j < s.n_per_conf) {
    const size_t i = (size_t)c * s.n_per_conf + j;
    const double im = s.inv_mass[i];
    if (im > 0.0) {
      double vx = s.v[3 * i + 0], vy = s.v[3 * i + 1], vz = s.v[3 * i + 2];
      if (!frozen && t > 0) {   // B(dt/2): v += dt/2 * a, a = -dE/dx / m in A / fs^2
        const double h = 0.5 * dt * s.accel * im;
        vx -= h * (double)a.grad[3 * i + 0];
        vy -= h * (double)a.grad[3 * i + 1];
        vz -= h * (double)a.grad[3 * i + 2];
        s.v[3 * i + 0] = vx;
        s.v[3 * i + 1] = vy;
        s.v[3 * i + 2] = vz;
      }
      ke = 0.5 * (vx * vx + vy * vy + vz * vz) / im;
      if (a.force_stdev) fmax_ = (double)a.force_stdev[i];
    }
  }
  block_reduce<1>(&ke, fmax_, sv, sw);
  if (threadIdx.x == 0) {
    double* p = s.partials + 2 * ((size_t)c * gridDim.x + blockIdx.x);
    p[0] = ke;
    p[1] = fmax_;
  }
}

// isotropic stochastic cell rescaling of conformer c at step t (Euler-Maruyama in eps = ln V), by thread 0 of every
// block of the conformer (the same inputs, so the same mu everywhere): tot = {sum 1/2 m v^2 (E_kin in amu A^2 / fs^2),
// -, tr W}; mu goes to tot[3], the float32-rounded new cell and its inverse to cell / inv.  Block 0 writes the master cell of step t + 1, the float32
// cell of the next force step, the record {V, P_int} of step t and the cell of step t's frame.
__device__ void rescale_cell(const MdArgs& a, int c, long long t, const double* par, double* tot, double* cell,
                             double* inv) {
  const ani_md_state& s = a.s;
  const ani_md_barostat& b = a.baro;
  const double* h = b.master + ((size_t)(t & 1) * s.n_conf + c) * 9;
  const double* bp = b.params + (size_t)c * ANI_MD_BARO_PARAMS;   // P0 (Hartree / A^3), tau_p (fs), beta_T (A^3 / Hartree)
  const double vol = fabs(det3(h));
  const double p_int = (2.0 * tot[0] / s.accel - tot[2]) / (3.0 * vol);
  const double kt = s.kb * par[1], dt = par[0], bt = bp[2] / bp[1];
  // (the k_B T / V term of the volume form, dV = -(beta_T V / tau_p)(P0 - P_int - k_B T / V) dt + ..., cancels against
  // the Ito correction of eps = ln V: keeping it here would sample V^(N+1) exp(-P0 V / k_B T), one power too many)
  const double de = -bt * (bp[0] - p_int) * dt + sqrt(2.0 * kt * bt * dt / vol) * md_normal(s.seed, t, c, 3);
  const double mu = exp(de / 3.0);
  tot[3] = mu;
  for (int k = 0; k < 9; ++k) cell[k] = (double)(float)(mu * h[k]);
  invert3(cell, inv);
  if (blockIdx.x != 0) return;
  double* hn = b.master + ((size_t)((t + 1) & 1) * s.n_conf + c) * 9;
  float* out = b.cell_out + (size_t)c * b.cell_stride;
  for (int k = 0; k < 9; ++k) {
    hn[k] = mu * h[k];
    out[k] = (float)(mu * h[k]);
  }
  double* rec = b.record + ((size_t)(t % s.thermo_rows) * s.n_conf + c) * ANI_MD_BARO;
  rec[0] = vol;
  rec[1] = p_int;
  if (s.record_every > 0 && t % s.record_every == 0) {
    double* fc = b.frame_cells + ((size_t)((t / s.record_every) % s.frame_slots) * s.n_conf + c) * 9;
    for (int k = 0; k < 9; ++k) fc[k] = h[k];
  }
}

// launch 2 of a step: totals, thermo, frame, stop check, (the cell rescaling,) and the move to x(t+1)
__global__ void __launch_bounds__(MD_BLOCK) k_md_start(const __grid_constant__ MdArgs a) {
  __shared__ double cell[9], inv[9], tot[4];
  const ani_md_state& s = a.s;
  const bool npt = a.baro.master != nullptr;
  const int c = blockIdx.y, j = blockIdx.x * MD_BLOCK + threadIdx.x, nb = gridDim.x;
  const long long t = s.counter[1];
  const double* par = s.params + (size_t)c * ANI_MD_PARAMS;
  if (threadIdx.x < 32) {   // the conformer's {E_kin, max force stdev}, by warp_reduce of its partials
    const double* p = s.partials + 2 * (size_t)c * nb;
    double r[2];
    warp_reduce<1, 1>(threadIdx.x, nb, [&](int b, double* v) {
      v[0] = p[2 * b];
      v[1] = p[2 * b + 1];
    }, r);
    if (threadIdx.x == 0) {
      tot[0] = r[0];
      tot[1] = r[1];
    }
  } else if (npt && threadIdx.x < 64) {   // the trace of the conformer's virial slots, in the same fixed order
    const double* w = a.baro.virial + (size_t)c * a.baro.virial_slots * 9;
    double tr;
    warp_reduce<1, 0>(threadIdx.x - 32, a.baro.virial_slots, [&](int k, double* v) {
      v[0] = w[9 * k] + w[9 * k + 4] + w[9 * k + 8];
    }, &tr);
    if (threadIdx.x == 32) tot[2] = tr;
  }
  if (npt) {
    __syncthreads();
    if (threadIdx.x == 0) rescale_cell(a, c, t, par, tot, cell, inv);
  } else {
    load_cell(a.cells, a.cell_stride, c, cell, inv);
  }
  __syncthreads();
  // stop_step[c] is written below by block 0 of this conformer only, and only with the value t: a block that reads it
  // concurrently sees -1 or t, and "stopped before this step" is false for both
  const long long ss = s.stop_step[c];
  const bool stopped_before = ss >= 0 && ss < t;
  const bool trip = !stopped_before && a.qbc && (a.qbc[c] > par[3] || tot[1] > par[4]);
  const bool frozen = stopped_before || trip;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const double ekin = tot[0] / s.accel;   // amu A^2 / fs^2 -> Hartree
    double* row = s.thermo + ((size_t)(t % s.thermo_rows) * s.n_conf + c) * ANI_MD_THERMO;
    row[0] = (double)t;
    row[1] = a.energies[c];
    row[2] = ekin;
    row[3] = 2.0 * ekin / (par[5] * s.kb);   // par[5] = 3 N_real
    if (trip) s.stop_step[c] = t;
    if (c == 0) s.counter[0] = t + 1;
  }
  if (j >= s.n_per_conf) return;
  const size_t n = (size_t)s.n_conf * s.n_per_conf, i = (size_t)c * s.n_per_conf + j;
  double x = s.x[3 * i + 0], y = s.x[3 * i + 1], z = s.x[3 * i + 2];
  double vx = s.v[3 * i + 0], vy = s.v[3 * i + 1], vz = s.v[3 * i + 2];
  if (s.record_every > 0 && t % s.record_every == 0) {
    double* f = s.frames + (size_t)((t / s.record_every) % s.frame_slots) * (1 + s.frame_velocities) * 3 * n;
    f[3 * i + 0] = x;
    f[3 * i + 1] = y;
    f[3 * i + 2] = z;
    if (s.frame_velocities) {
      f[3 * (n + i) + 0] = vx;
      f[3 * (n + i) + 1] = vy;
      f[3 * (n + i) + 2] = vz;
    }
  }
  if (trip && s.trigger) {
    s.trigger[3 * i + 0] = x;
    s.trigger[3 * i + 1] = y;
    s.trigger[3 * i + 2] = z;
    s.trigger[3 * (n + i) + 0] = vx;
    s.trigger[3 * (n + i) + 1] = vy;
    s.trigger[3 * (n + i) + 2] = vz;
  }
  const double im = s.inv_mass[i];
  if (frozen || !(im > 0.0)) return;
  const double dt = par[0];
  const double h = 0.5 * dt * s.accel * im;
  vx -= h * (double)a.grad[3 * i + 0];   // B(dt/2)
  vy -= h * (double)a.grad[3 * i + 1];
  vz -= h * (double)a.grad[3 * i + 2];
  if (s.integrator == ANI_MD_VERLET) {   // A(dt)
    x += dt * vx;
    y += dt * vy;
    z += dt * vz;
  } else {   // A(dt/2) O(dt) A(dt/2)
    const double hd = 0.5 * dt;
    x += hd * vx;
    y += hd * vy;
    z += hd * vz;
    const double cf = exp(-par[2] * dt);
    const double sg = sqrt((1.0 - cf * cf) * s.kb * par[1] * s.accel * im);   // sqrt((1 - c^2) kT / m) in A / fs
    const int g = (int)i;
    vx = cf * vx + sg * md_normal(s.seed, t, g, 0);
    vy = cf * vy + sg * md_normal(s.seed, t, g, 1);
    vz = cf * vz + sg * md_normal(s.seed, t, g, 2);
    x += hd * vx;
    y += hd * vy;
    z += hd * vz;
  }
  if (npt) {   // x(t+1) = mu x', v / mu
    const double mu = tot[3];
    x *= mu;
    y *= mu;
    z *= mu;
    vx /= mu;
    vy /= mu;
    vz /= mu;
  }
  s.x[3 * i + 0] = x;
  s.x[3 * i + 1] = y;
  s.x[3 * i + 2] = z;
  s.v[3 * i + 0] = vx;
  s.v[3 * i + 1] = vy;
  s.v[3 * i + 2] = vz;
  write_coords(a.coords, i, x, y, z, npt || a.cells, cell, inv);
}

// one CTA per conformer: optional removal of the centre-of-mass momentum, then the coordinates of step 0
__global__ void __launch_bounds__(MD_BLOCK) k_md_init(const __grid_constant__ MdArgs a) {
  __shared__ double sv[MD_BLOCK], sw[MD_BLOCK], tot[4];
  const ani_md_state& s = a.s;
  const int c = blockIdx.x, A = s.n_per_conf;
  const size_t base = (size_t)c * A;
  if (a.reset) {
    for (int k = 0; k < 4; ++k) {   // the momentum components sum m v_k, then the total mass
      double p = 0.0, unused = 0.0;
      for (int j = threadIdx.x; j < A; j += MD_BLOCK) {
        const double im = s.inv_mass[base + j];
        if (im > 0.0) p += (k < 3 ? s.v[3 * (base + j) + k] : 1.0) / im;
      }
      block_reduce<1>(&p, unused, sv, sw);
      if (threadIdx.x == 0) tot[k] = p;
      __syncthreads();   // (sv is reused by the next reduction)
    }
    for (int j = threadIdx.x; j < A; j += MD_BLOCK) {
      if (s.inv_mass[base + j] > 0.0)
        for (int k = 0; k < 3; ++k) s.v[3 * (base + j) + k] -= tot[k] / tot[3];
    }
  }
  conformer_coords(a, c, A, s.x);
}

__global__ void __launch_bounds__(MD_BLOCK) k_md_noise(unsigned long long seed, long long step, int n, double* out) {
  const int i = blockIdx.x * MD_BLOCK + threadIdx.x;
  if (i >= n) return;
  for (int k = 0; k < 3; ++k) out[3 * (size_t)i + k] = md_normal(seed, step, i, k);
}

__global__ void __launch_bounds__(MD_BLOCK) k_md_cell_noise(unsigned long long seed, long long step, int n, double* out) {
  const int c = blockIdx.x * MD_BLOCK + threadIdx.x;
  if (c < n) out[c] = md_normal(seed, step, c, 3);
}

bool md_state_ok(const ani_md_state* s) {
  return s && s->x && s->v && s->inv_mass && s->n_conf >= 1 && s->n_per_conf >= 1;
}

int md_step(const ani_md_state* s, const float* grad, const double* energies, const double* qbc,
            const float* force_stdev, const float* cells, int cell_stride, float* coords, void* stream,
            const ani_md_barostat* baro = nullptr) {
  if (!md_state_ok(s) || !s->params || !s->counter || !s->stop_step || !s->thermo || !s->partials) return ANI_ERR_BAD_ARG;
  if (!grad || !energies || !coords || (!qbc != !force_stdev)) return ANI_ERR_BAD_ARG;
  if ((s->integrator != ANI_MD_VERLET && s->integrator != ANI_MD_LANGEVIN) || s->thermo_rows < 1) return ANI_ERR_BAD_ARG;
  if (s->record_every < 0 || (s->record_every > 0 && (!s->frames || s->frame_slots < 1))) return ANI_ERR_BAD_ARG;
  if (!(s->accel > 0.0) || !(s->kb > 0.0)) return ANI_ERR_BAD_ARG;
  const int rc = launch_shape(s->n_conf, s->n_per_conf);
  if (rc != ANI_OK) return rc;
  MdArgs a = {{grad, energies, cells, cell_stride, coords, 0}, *s, qbc, force_stdev, baro ? *baro : ani_md_barostat{}};
  const dim3 grid((s->n_per_conf + MD_BLOCK - 1) / MD_BLOCK, s->n_conf);
  cudaStream_t st = (cudaStream_t)stream;
  k_md_finish<<<grid, MD_BLOCK, 0, st>>>(a);
  k_md_start<<<grid, MD_BLOCK, 0, st>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

}  // namespace ani

using namespace ani;

extern "C" int ani_b200_md_init(const ani_md_state* state, const float* cells, int cell_mode, int zero_momentum,
                                float* coords, void* stream) {
  MdArgs a = {};
  if (!md_state_ok(state) || !coords || !init_cells(a, cells, cell_mode)) return ANI_ERR_BAD_ARG;
  a.s = *state;
  a.coords = coords;
  a.reset = zero_momentum != 0;
  k_md_init<<<state->n_conf, MD_BLOCK, 0, (cudaStream_t)stream>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_md_step(const ani_md_state* state, const float* grad, const double* energies,
                                const double* qbc, const float* force_stdev, const float* cell, float* coords,
                                void* stream) {
  return md_step(state, grad, energies, qbc, force_stdev, cell, 0, coords, stream);
}

extern "C" int ani_b200_md_step_cells(const ani_md_state* state, const float* grad, const double* energies,
                                      const double* qbc, const float* force_stdev, const float* lattice,
                                      float* coords, void* stream) {
  if (!lattice) return ANI_ERR_BAD_ARG;
  return md_step(state, grad, energies, qbc, force_stdev, lattice, ANI_LATTICE_STRIDE, coords, stream);
}

extern "C" int ani_b200_md_step_npt(const ani_md_state* state, const ani_md_barostat* baro, const float* grad,
                                    const double* energies, float* coords, void* stream) {
  if (!md_state_ok(state) || !baro || state->integrator != ANI_MD_LANGEVIN) return ANI_ERR_BAD_ARG;
  const ani_md_barostat& b = *baro;
  if (!b.master || !b.params || !b.cell_out || !b.virial || !b.record || b.cell_stride < 9 || b.virial_slots < 1)
    return ANI_ERR_BAD_ARG;
  if (state->record_every > 0 && !b.frame_cells) return ANI_ERR_BAD_ARG;
  return md_step(state, grad, energies, nullptr, nullptr, nullptr, 0, coords, stream, baro);
}

extern "C" int ani_b200_md_noise(unsigned long long seed, long long step, int n, double* out, void* stream) {
  if (n < 1 || !out) return ANI_ERR_BAD_ARG;
  k_md_noise<<<(n + MD_BLOCK - 1) / MD_BLOCK, MD_BLOCK, 0, (cudaStream_t)stream>>>(seed, step, n, out);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_md_cell_noise(unsigned long long seed, long long step, int n_conf, double* out, void* stream) {
  if (n_conf < 1 || !out) return ANI_ERR_BAD_ARG;
  k_md_cell_noise<<<(n_conf + MD_BLOCK - 1) / MD_BLOCK, MD_BLOCK, 0, (cudaStream_t)stream>>>(seed, step, n_conf, out);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}
