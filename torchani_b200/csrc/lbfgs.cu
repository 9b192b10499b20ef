// Geometry optimisation on the device: L-BFGS as ASE's ase.optimize.LBFGS defines it (without its line search), one
// independent optimisation per conformer.  The positions, the last step's positions and gradient, and a ring of the
// last `memory` pairs s = x(t) - x(t-1), y = g(t) - g(t-1) (float64) stay in device memory with the slot-indexed
// products s_i.y_j and y_i.y_j, so K whole steps (L-BFGS + force step) capture into one CUDA graph, as FIRE's (opt.cu).
//
// The direction p = -H g is not formed by the two-loop recursion (2L dependent conformer-wide dot products) but by the
// compact representation of the same L-pair inverse BFGS matrix (Byrd, Nocedal & Schnabel, Math. Prog. 63 (1994),
// Thm 2.2): with S, Y the live pairs in chronological order, R the upper triangle of S^T Y, D = diag(s_i.y_i),
// u = S^T g, w = Y^T g and H0 = 1 / alpha,
//     r = R^-1 u,   a = R^-T ((D + H0 Y^T Y) r - H0 w),   b = -H0 r,   p = -(H0 g + S a + Y b).
// It needs only s_i.y_i != 0, so it holds for pairs of negative curvature too.
//
// One step is the force step at x(t) followed by four launches (ani_b200_lbfgs_step):
//   k_lbfgs_dots       grid (tiles of LB_TILE atoms, groups of LB_ROWS rows, conformers): f, g and (k >= 1) the new
//                      pair of the block's atoms; blocks of group 0 write the pair to ring slot head % (memory + 1) and
//                      the tile's largest |f_i|^2; warp w of group q forms the tile's partial sums {s.g, y.g, s.y_new,
//                      y.y_new} of row 8 q + w: rows 0..L-1 are the live pairs (chronological), row L the new pair
//   k_lbfgs_solve      one block per conformer: the partials summed over the tiles in order, the record, the
//                      convergence check, the new pair's column of SY and YY (or the pair skipped when y.s == 0), the
//                      two triangular solves on R in shared memory, and a, b, k + 1 and the new ring head
//   k_lbfgs_direction  per tile of LB_TILE atoms: p = -(H0 g + sum_j a_j s_j + b_j y_j), the slots split over the
//                      block's 8 warps and their sums added in warp order; per block the largest |p_i|^2
//   k_lbfgs_move       per atom: the conformer's largest |p_i| from the direction partials (in order), the clamp
//                      p min(1, maxstep / max_i |p_i|) (applied when max_i |p_i| >= maxstep), the damping, x_prev = x,
//                      g_prev = g, x(t+1) and its float32 coordinates wrapped into the cell
// The ring has memory + 1 slots: the dot sweep writes the new pair before the solve knows whether y.s == 0, and the
// spare slot keeps the oldest live pair intact until then (a skipped pair leaves no gap).  Race rules: every launch
// reads only what an earlier launch wrote, except the dot sweep's ring slot head % (memory + 1), which no live row
// reads, and conv_step, SY, YY and the conformer's {k, head}, which only the conformer's solve block touches.  Every
// sum is float64 in a fixed order without atomics: the same state and forces give the same bits.  The step counter
// lives on the device with the protocol of md.cu (the dot sweep copies counter[0] to counter[1], the solve writes
// counter[0] = t + 1).
#include "md_common.cuh"

namespace ani {

constexpr int LB_THREADS = 256;                  // threads of the dot-sweep, direction and move blocks
constexpr int LB_TILE = ANI_LBFGS_TILE;          // atoms per dot-sweep tile and per direction block (<= 32)
constexpr int LB_ROWS = LB_THREADS / ANI_WARP;   // rows per dot-sweep block: one warp each
constexpr int LB_SOLVE = 128;                    // threads of a solve block

struct LbfgsArgs : LoopArgs {
  ani_lbfgs_state s;
};

__device__ __forceinline__ int ring_slots(const ani_lbfgs_state& s) { return s.memory + 1; }
__device__ __forceinline__ int n_tiles(const ani_lbfgs_state& s) { return (s.n_per_conf + LB_TILE - 1) / LB_TILE; }

// ring slot `slot` of conformer c: f64[n_per_conf][3]
__device__ __forceinline__ size_t ring_at(const ani_lbfgs_state& s, int c, int slot) {
  return ((size_t)c * ring_slots(s) + slot) * 3 * s.n_per_conf;
}

// scratch: dot partials f64[n_conf][tiles][memory + 1][4], then the tiles' largest |f_i|^2 f64[n_conf][tiles], then the
// direction blocks' largest |p_i|^2 f64[n_conf][tiles]
__device__ __forceinline__ double* dot_partials(const ani_lbfgs_state& s, int c, int tile) {
  return s.partials + ((size_t)c * n_tiles(s) + tile) * ring_slots(s) * 4;
}
__device__ __forceinline__ double* fmax_partials(const ani_lbfgs_state& s, int c) {
  return s.partials + (size_t)s.n_conf * n_tiles(s) * ring_slots(s) * 4 + (size_t)c * n_tiles(s);
}
__device__ __forceinline__ double* pmax_partials(const ani_lbfgs_state& s, int c) {
  return fmax_partials(s, s.n_conf) + (size_t)c * n_tiles(s);
}

// g = dE/dx * force_scale of atom i (eV / A; f = -g, and 0 for fixed and padding atoms)
__device__ __forceinline__ void grad_of(const LbfgsArgs& a, size_t i, double* g) {
  const double fs = a.s.force_scale[i];
  g[0] = (double)a.grad[3 * i + 0] * fs;
  g[1] = (double)a.grad[3 * i + 1] * fs;
  g[2] = (double)a.grad[3 * i + 2] * fs;
}

// launch 1: the new pair and the dot products of every row with g and y_new, per tile of atoms (see the file comment)
__global__ void __launch_bounds__(LB_THREADS) k_lbfgs_dots(const __grid_constant__ LbfgsArgs a) {
  __shared__ double sg[3 * LB_TILE], ss[3 * LB_TILE], sy[3 * LB_TILE], wmax[LB_TILE / ANI_WARP];
  const ani_lbfgs_state& s = a.s;
  const int tile = blockIdx.x, grp = blockIdx.y, c = blockIdx.z, lane = threadIdx.x % ANI_WARP;
  if (tile == 0 && grp == 0 && c == 0 && threadIdx.x == 0) s.counter[1] = s.counter[0];
  const long long k = s.iter[2 * c], head = s.iter[2 * c + 1];
  const bool frozen = s.conv_step[c] >= 0;   // converged at an earlier step (the solve of this step writes it)
  const int M = ring_slots(s);
  const int nold = (int)min((long long)s.memory, head);
  const int rows = frozen ? 0 : nold + (k >= 1 ? 1 : 0);
  if (grp > 0 && grp * LB_ROWS >= rows) return;   // a block without rows (group 0 always writes the fmax partial)
  const int a0 = tile * LB_TILE, na = min(LB_TILE, s.n_per_conf - a0);
  if (threadIdx.x < LB_TILE) {
    double f2 = 0.0;
    if ((int)threadIdx.x < na) {
      const size_t i = (size_t)c * s.n_per_conf + a0 + threadIdx.x;
      double g[3];
      grad_of(a, i, g);
      f2 = g[0] * g[0] + g[1] * g[1] + g[2] * g[2];
      const bool pair = k >= 1 && !frozen;
      double* rs = s.s + ring_at(s, c, (int)(head % M)) + 3 * (size_t)(a0 + threadIdx.x);
      double* ry = s.y + ring_at(s, c, (int)(head % M)) + 3 * (size_t)(a0 + threadIdx.x);
      for (int d = 0; d < 3; ++d) {
        const int e = 3 * threadIdx.x + d;
        sg[e] = g[d];
        if (pair) {
          ss[e] = s.x[3 * i + d] - s.x_prev[3 * i + d];
          sy[e] = g[d] - s.g_prev[3 * i + d];
          if (grp == 0) {
            rs[d] = ss[e];
            ry[d] = sy[e];
          }
        }
      }
    }
    if (grp == 0) {
      warp_tree<0, 1>(&f2);
      if (lane == 0) wmax[threadIdx.x / ANI_WARP] = f2;
    }
  }
  __syncthreads();
  if (grp == 0 && threadIdx.x == 0) {
    double m = wmax[0];
    for (int w = 1; w < LB_TILE / ANI_WARP; ++w) m = fmax(m, wmax[w]);
    fmax_partials(s, c)[tile] = m;
  }
  const int r = grp * LB_ROWS + threadIdx.x / ANI_WARP;
  if (r >= rows) return;
  const double *vs = ss, *vy = sy;   // row nold: the new pair, from shared memory (its ring slot is being written)
  if (r < nold) {
    const int slot = (int)((head - nold + r) % M);
    vs = s.s + ring_at(s, c, slot) + 3 * (size_t)a0;
    vy = s.y + ring_at(s, c, slot) + 3 * (size_t)a0;
  }
  double d[4] = {0.0, 0.0, 0.0, 0.0};
  for (int e = lane; e < 3 * na; e += ANI_WARP) {
    const double se = vs[e], ye = vy[e];
    d[0] += se * sg[e];
    d[1] += ye * sg[e];
    if (k >= 1) {
      d[2] += se * sy[e];
      d[3] += ye * sy[e];
    }
  }
  warp_tree<4, 0>(d);
  if (lane == 0) {
    double* out = dot_partials(s, c, tile) + 4 * r;
    for (int q = 0; q < 4; ++q) out[q] = d[q];
  }
}

// launch 2: one block per conformer (see the file comment); dynamic shared memory: R f64[memory][memory], then the
// row totals f64[4][memory + 1], r, a and 1 / R_ii f64[memory] each and the live slots i32[memory].  The triangular
// solves run on warp 0 in the column (axpy) form, one dependent step per pair, each v_j updated in a fixed order.
__global__ void __launch_bounds__(LB_SOLVE) k_lbfgs_solve(const __grid_constant__ LbfgsArgs a) {
  extern __shared__ double sm[];
  __shared__ int flag;
  const ani_lbfgs_state& s = a.s;
  const int c = blockIdx.x, M = ring_slots(s), mem = s.memory, nt = n_tiles(s);
  double* R = sm;
  double* tot = R + (size_t)mem * mem;   // {u, w, s.y_new, y.y_new} of each row
  double* rv = tot + 4 * M;   // u, then r
  double* av = rv + mem;      // t, then a
  double* dinv = av + mem;
  int* slot = (int*)(dinv + mem);
  const long long t = s.counter[1], k = s.iter[2 * c], head = s.iter[2 * c + 1];
  const double* par = s.params + (size_t)c * ANI_LBFGS_PARAMS;   // maxstep, damping, H0, fmax
  const double h0 = par[2];
  if (threadIdx.x < ANI_WARP) {   // fmax(t): warp_reduce of the tiles' maxima
    const double* fp = fmax_partials(s, c);
    double m;
    warp_reduce<0, 1>(threadIdx.x, nt, [&](int b, double* v) { v[0] = fp[b]; }, &m);
    if (threadIdx.x == 0) {
      const double fm = sqrt(m);
      double* row = s.record + ((size_t)(t % s.record_rows) * s.n_conf + c) * ANI_LBFGS_RECORD;
      row[0] = (double)t;
      row[1] = a.energies[c];
      row[2] = fm;
      const bool before = s.conv_step[c] >= 0;
      const bool conv = !before && fm < par[3];
      if (conv) s.conv_step[c] = t;
      if (c == 0) s.counter[0] = t + 1;
      flag = before || conv;
    }
  }
  __syncthreads();
  if (flag) return;   // converged: nothing of this conformer changes again
  const int nold = (int)min((long long)mem, head);
  const int rows = nold + (k >= 1 ? 1 : 0);
  for (int r = threadIdx.x; r < rows; r += LB_SOLVE) {   // the row totals, summed over the tiles in order
    double q[4] = {0.0, 0.0, 0.0, 0.0};
    for (int b = 0; b < nt; ++b) {
      const double* p = dot_partials(s, c, b) + 4 * r;
      for (int j = 0; j < 4; ++j) q[j] += p[j];
    }
    for (int j = 0; j < 4; ++j) tot[j * M + r] = q[j];
  }
  __syncthreads();
  // the new pair (row nold) joins the history unless y.s == 0 (ASE would divide by zero there)
  const int keep = (k >= 1 && tot[2 * M + nold] != 0.0) ? 1 : 0;
  const long long nhead = head + keep;
  const int L = (int)min((long long)mem, nhead);
  const int drop = nold + keep - L;            // 1 when the oldest pair leaves a full history
  const int nslot = (int)(head % M);
  double* SY = s.sy + (size_t)c * M * M;
  double* YY = s.yy + (size_t)c * M * M;
  if (keep) {   // column nslot of SY (s_i.y_new, upper triangle only) and of YY (symmetric)
    for (int r = drop + threadIdx.x; r <= nold; r += LB_SOLVE) {
      const int sl = r < nold ? (int)((head - nold + r) % M) : nslot;
      SY[(size_t)sl * M + nslot] = tot[2 * M + r];
      YY[(size_t)sl * M + nslot] = tot[3 * M + r];
      YY[(size_t)nslot * M + sl] = tot[3 * M + r];
    }
  }
  __syncthreads();
  // chronological pair j of the L live ones: row drop + j, ring slot (nhead - L + j) % M
  for (int j = threadIdx.x; j < L; j += LB_SOLVE) slot[j] = (int)((nhead - L + j) % M);
  __syncthreads();
  for (int idx = threadIdx.x; idx < L * L; idx += LB_SOLVE) {
    const int i = idx / L, j = idx % L;
    R[idx] = i <= j ? SY[(size_t)slot[i] * M + slot[j]] : 0.0;
  }
  for (int j = threadIdx.x; j < L; j += LB_SOLVE) rv[j] = tot[drop + j];
  __syncthreads();
  for (int j = threadIdx.x; j < L; j += LB_SOLVE) dinv[j] = 1.0 / R[j * L + j];
  __syncthreads();
  if (threadIdx.x < ANI_WARP) {   // r = R^-1 u by columns: r_i = v_i / R_ii, then v_j -= R_ji r_i for j < i
    for (int i = L - 1; i >= 0; --i) {
      const double ri = rv[i] * dinv[i];
      for (int j = threadIdx.x; j < i; j += ANI_WARP) rv[j] -= R[j * L + i] * ri;
      __syncwarp();
      if (threadIdx.x == 0) rv[i] = ri;
      __syncwarp();
    }
  }
  __syncthreads();
  for (int i = threadIdx.x / ANI_WARP; i < L; i += LB_SOLVE / ANI_WARP) {   // t = (D + H0 Y^T Y) r - H0 w, a warp a row
    const double* yrow = YY + (size_t)slot[i] * M;
    double acc = 0.0;
    for (int j = threadIdx.x % ANI_WARP; j < L; j += ANI_WARP) acc += yrow[slot[j]] * rv[j];
    warp_tree<1, 0>(&acc);
    acc = __shfl_sync(ANI_FULL_MASK, acc, 0);   // (to every lane: the row loop compiles shorter than for lane 0 only)
    if (threadIdx.x % ANI_WARP == 0) av[i] = R[i * L + i] * rv[i] + h0 * acc - h0 * tot[M + drop + i];
  }
  __syncthreads();
  if (threadIdx.x < ANI_WARP) {   // a = R^-T t by rows: a_i = v_i / R_ii, then v_j -= R_ij a_i for j > i
    for (int i = 0; i < L; ++i) {
      const double ai = av[i] * dinv[i];
      for (int j = i + 1 + threadIdx.x; j < L; j += ANI_WARP) av[j] -= R[i * L + j] * ai;
      __syncwarp();
      if (threadIdx.x == 0) av[i] = ai;
      __syncwarp();
    }
  }
  __syncthreads();
  double* coef = s.coef + (size_t)c * 2 * mem;
  for (int i = threadIdx.x; i < L; i += LB_SOLVE) {
    coef[i] = av[i];
    coef[mem + i] = -h0 * rv[i];
  }
  if (threadIdx.x == 0) {
    s.iter[2 * c] = k + 1;
    s.iter[2 * c + 1] = nhead;
  }
}

// launch 3: p = -(H0 g + sum_j (a_j s_j + b_j y_j)) per tile of LB_TILE atoms: warp w sums the slots j = w, w + 8, ...
// (chronological) for the tile's 3 LB_TILE elements, lane-strided, and the warps' sums are added to H0 g in warp order;
// per block the largest |p_i|^2
__global__ void __launch_bounds__(LB_THREADS) k_lbfgs_direction(const __grid_constant__ LbfgsArgs a) {
  __shared__ double ca[ANI_LBFGS_MAX_MEMORY], cb[ANI_LBFGS_MAX_MEMORY], part[LB_ROWS][3 * LB_TILE];
  __shared__ int slot[ANI_LBFGS_MAX_MEMORY];
  const ani_lbfgs_state& s = a.s;
  const int c = blockIdx.y, a0 = blockIdx.x * LB_TILE, M = ring_slots(s);
  const int na = min(LB_TILE, s.n_per_conf - a0), w = threadIdx.x / ANI_WARP, lane = threadIdx.x % ANI_WARP;
  if (s.conv_step[c] >= 0) return;   // frozen: the move reads nothing of this conformer
  const long long head = s.iter[2 * c + 1];
  const int L = (int)min((long long)s.memory, head);
  const double* coef = s.coef + (size_t)c * 2 * s.memory;
  for (int q = threadIdx.x; q < L; q += LB_THREADS) {
    ca[q] = coef[q];
    cb[q] = coef[s.memory + q];
    slot[q] = (int)((head - L + q) % M);
  }
  __syncthreads();
  double z[3 * LB_TILE / ANI_WARP];
#pragma unroll
  for (int m = 0; m < 3 * LB_TILE / ANI_WARP; ++m) z[m] = 0.0;
  for (int q = w; q < L; q += LB_ROWS) {
    const double* rs = s.s + ring_at(s, c, slot[q]) + 3 * (size_t)a0;
    const double* ry = s.y + ring_at(s, c, slot[q]) + 3 * (size_t)a0;
    const double aq = ca[q], bq = cb[q];
#pragma unroll
    for (int m = 0; m < 3 * LB_TILE / ANI_WARP; ++m) {
      const int e = lane + m * ANI_WARP;
      if (e < 3 * na) {
        z[m] += aq * rs[e];
        z[m] += bq * ry[e];
      }
    }
  }
#pragma unroll
  for (int m = 0; m < 3 * LB_TILE / ANI_WARP; ++m) part[w][lane + m * ANI_WARP] = z[m];
  __syncthreads();
  if (threadIdx.x < 3 * LB_TILE) {
    const int e = threadIdx.x;
    double v = 0.0;
    if (e < 3 * na) {
      const size_t i = ((size_t)c * s.n_per_conf + a0) * 3 + e;
      v = s.params[(size_t)c * ANI_LBFGS_PARAMS + 2] * ((double)a.grad[i] * s.force_scale[i / 3]);
      for (int q = 0; q < LB_ROWS; ++q) v += part[q][e];
      s.p[i] = -v;
    }
    part[0][e] = v;   // (row 0 of part is read by this thread only before)
  }
  __syncthreads();
  if (threadIdx.x < ANI_WARP) {
    double p2 = 0.0;
    if ((int)threadIdx.x < na) {
      const double* v = part[0] + 3 * threadIdx.x;
      p2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    }
    warp_tree<0, 1>(&p2);
    if (threadIdx.x == 0) pmax_partials(s, c)[blockIdx.x] = p2;
  }
}

// launch 4: the clamp and damping of the conformer's step, x_prev = x, g_prev = g, x(t+1) and its float32 coordinates
__global__ void __launch_bounds__(LB_THREADS) k_lbfgs_move(const __grid_constant__ LbfgsArgs a) {
  __shared__ double cell[9], inv[9], scale;
  const ani_lbfgs_state& s = a.s;
  const int c = blockIdx.y, j = blockIdx.x * LB_THREADS + threadIdx.x;
  if (s.conv_step[c] >= 0) return;   // converged at this step or before: nothing moves
  if (threadIdx.x < ANI_WARP) {   // max_i |p_i|^2: warp_reduce of the direction blocks' maxima
    const double* pp = pmax_partials(s, c);
    double m;
    warp_reduce<0, 1>(threadIdx.x, n_tiles(s), [&](int b, double* v) { v[0] = pp[b]; }, &m);
    if (threadIdx.x == 0) {
      const double maxstep = s.params[(size_t)c * ANI_LBFGS_PARAMS], longest = sqrt(m);
      scale = longest >= maxstep ? maxstep / longest : 1.0;   // ASE's determine_step: the longest atom step
    }
  }
  load_cell(a.cells, a.cell_stride, c, cell, inv);
  __syncthreads();
  if (j >= s.n_per_conf) return;
  const size_t i = (size_t)c * s.n_per_conf + j;
  if (s.force_scale[i] == 0.0) return;   // fixed and padding atoms: g = s = y = 0, so p = 0 and x never moves
  const double damping = s.params[(size_t)c * ANI_LBFGS_PARAMS + 1];
  double g[3], x[3];
  grad_of(a, i, g);
  for (int d = 0; d < 3; ++d) {
    const double x0 = s.x[3 * i + d];
    x[d] = x0 + s.p[3 * i + d] * scale * damping;
    s.x_prev[3 * i + d] = x0;
    s.g_prev[3 * i + d] = g[d];
    s.x[3 * i + d] = x[d];
  }
  write_coords(a.coords, i, x[0], x[1], x[2], a.cells, cell, inv);
}

// one CTA per conformer: with reset, x_prev = x, g_prev = 0 and {k, head} = {0, 0}; then the coordinates of x
__global__ void __launch_bounds__(LB_THREADS) k_lbfgs_init(const __grid_constant__ LbfgsArgs a) {
  const ani_lbfgs_state& s = a.s;
  const int c = blockIdx.x, A = s.n_per_conf;
  const size_t base = (size_t)c * A;
  if (a.reset) {
    for (int j = threadIdx.x; j < 3 * A; j += LB_THREADS) {
      s.x_prev[3 * base + j] = s.x[3 * base + j];
      s.g_prev[3 * base + j] = 0.0;
    }
    if (threadIdx.x == 0) {
      s.iter[2 * c] = 0;
      s.iter[2 * c + 1] = 0;
    }
  }
  conformer_coords(a, c, A, s.x);
}

size_t solve_smem(int memory) {
  return ((size_t)memory * memory + 4 * (memory + 1) + 3 * memory) * sizeof(double) + memory * sizeof(int);
}

bool lbfgs_state_ok(const ani_lbfgs_state* s) {
  return s && s->x && s->x_prev && s->g_prev && s->s && s->y && s->sy && s->yy && s->coef && s->p && s->iter &&
         s->force_scale && s->params && s->counter && s->n_conf >= 1 && s->n_per_conf >= 1 && s->memory >= 1 &&
         s->memory <= ANI_LBFGS_MAX_MEMORY;
}

int lbfgs_step(const ani_lbfgs_state* s, const float* grad, const double* energies, const float* cells,
               int cell_stride, float* coords, void* stream) {
  if (!lbfgs_state_ok(s) || !s->conv_step || !s->record || !s->partials || s->record_rows < 1) return ANI_ERR_BAD_ARG;
  if (!grad || !energies || !coords) return ANI_ERR_BAD_ARG;
  const int rc = launch_shape(s->n_conf, s->n_per_conf);
  if (rc != ANI_OK) return rc;
  const LbfgsArgs a = {{grad, energies, cells, cell_stride, coords, 0}, *s};
  const int tiles = (s->n_per_conf + LB_TILE - 1) / LB_TILE, groups = (s->memory + 1 + LB_ROWS - 1) / LB_ROWS;
  const size_t smem = solve_smem(s->memory);
  if (cudaFuncSetAttribute(k_lbfgs_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return ANI_ERR_CUDA;
  cudaStream_t st = (cudaStream_t)stream;
  k_lbfgs_dots<<<dim3(tiles, groups, s->n_conf), LB_THREADS, 0, st>>>(a);
  k_lbfgs_solve<<<s->n_conf, LB_SOLVE, smem, st>>>(a);
  k_lbfgs_direction<<<dim3(tiles, s->n_conf), LB_THREADS, 0, st>>>(a);
  k_lbfgs_move<<<dim3((s->n_per_conf + LB_THREADS - 1) / LB_THREADS, s->n_conf), LB_THREADS, 0, st>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

}  // namespace ani

using namespace ani;

extern "C" int ani_b200_lbfgs_init(const ani_lbfgs_state* state, const float* cells, int cell_mode, int reset,
                                   float* coords, void* stream) {
  LbfgsArgs a = {};
  if (!lbfgs_state_ok(state) || !coords || !init_cells(a, cells, cell_mode)) return ANI_ERR_BAD_ARG;
  a.s = *state;
  a.coords = coords;
  a.reset = reset != 0;
  k_lbfgs_init<<<state->n_conf, LB_THREADS, 0, (cudaStream_t)stream>>>(a);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_lbfgs_step(const ani_lbfgs_state* state, const float* grad, const double* energies,
                                   const float* cell, float* coords, void* stream) {
  return lbfgs_step(state, grad, energies, cell, 0, coords, stream);
}

extern "C" int ani_b200_lbfgs_step_cells(const ani_lbfgs_state* state, const float* grad, const double* energies,
                                         const float* lattice, float* coords, void* stream) {
  if (!lattice) return ANI_ERR_BAD_ARG;
  return lbfgs_step(state, grad, energies, lattice, ANI_LATTICE_STRIDE, coords, stream);
}
