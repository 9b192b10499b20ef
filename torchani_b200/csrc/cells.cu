// Bucket grid construction: wrap atoms into the cell, assign buckets, stable counting sort,
// species-grouped row layout for the MLP.  Replaces the ATen op chain of
// neighbors.py:418-507,554-615 / csrc/cell_list.cpp:266-350 with five small sync-free kernels.
#include <stdlib.h>

#include "common.cuh"

namespace ani {

// inverse of the 3x3 cell in double (host-quality), rows of `cell` are lattice vectors
__device__ __forceinline__ void cell_inverse(const float* __restrict__ cell, double (&iv)[9]) {
  double c[9];
  for (int k = 0; k < 9; ++k) c[k] = (double)cell[k];
  double det = c[0] * (c[4] * c[8] - c[5] * c[7]) - c[1] * (c[3] * c[8] - c[5] * c[6]) +
               c[2] * (c[3] * c[7] - c[4] * c[6]);
  double id = 1.0 / det;
  iv[0] = (c[4] * c[8] - c[5] * c[7]) * id;
  iv[1] = (c[2] * c[7] - c[1] * c[8]) * id;
  iv[2] = (c[1] * c[5] - c[2] * c[4]) * id;
  iv[3] = (c[5] * c[6] - c[3] * c[8]) * id;
  iv[4] = (c[0] * c[8] - c[2] * c[6]) * id;
  iv[5] = (c[2] * c[3] - c[0] * c[5]) * id;
  iv[6] = (c[3] * c[7] - c[4] * c[6]) * id;
  iv[7] = (c[1] * c[6] - c[0] * c[7]) * id;
  iv[8] = (c[0] * c[4] - c[1] * c[3]) * id;
}

// buckets along lattice direction d: frac_d = r . inv[:, d]; planes frac_d = const are 1/|inv[:, d]| apart
__device__ __forceinline__ int cell_buckets(const double (&iv)[9], int d, float bucket) {
  double w = 1.0 / sqrt(iv[d] * iv[d] + iv[3 + d] * iv[3 + d] + iv[6 + d] * iv[6 + d]);
  return (int)floor(w / (double)bucket);
}

// respect the caller's bucket capacity (buckets may only get larger than the cutoff)
__device__ __forceinline__ void cap_dims(ani_grid& g, int cap) {
  while ((long long)g.dims[0] * g.dims[1] * g.dims[2] > (long long)cap) {
    int big = 0;
    if (g.dims[1] > g.dims[big]) big = 1;
    if (g.dims[2] > g.dims[big]) big = 2;
    g.dims[big] = max(1, g.dims[big] - max(1, g.dims[big] / 8));
  }
}

// The grid of one call (executed by one thread).  mode 0 + pbc: buckets from the perpendicular
// widths of the cell (>= 1 bucket per cutoff, neighbors.py:618-662 uses edge lengths; widths are
// the safe choice for triclinic cells).  mode 0 without pbc: bounding box of the real atoms.
// mode 2 (a periodic batch in one shared cell): every conformer gets the sub-grid a single system in
// that cell would get from a 1 / n_conf share of the bucket capacity; dims are per conformer, nbins
// counts the buckets of all of them (conformer-major: bucket c * nb + local).
// (mode 3, one cell per conformer, needs every conformer's cell: conformer_lattices below)
__device__ ani_grid compute_grid(int n_conf, int n_per_conf, const float* __restrict__ cell, int pbc, int mode,
                                 float cutoff, int max_bins, const float* box_min, const float* box_max,
                                 int32_t* __restrict__ status) {
  ani_grid g;
  for (int k = 0; k < 9; ++k) g.cell[k] = g.inv[k] = 0.f;
  g.origin[0] = g.origin[1] = g.origin[2] = 0.f;
  g.dims[0] = g.dims[1] = g.dims[2] = 1;
  g.pbc = pbc;
  g.mode = mode;
  g.n_per_conf = n_per_conf;
  g.n_real = 0;
  const float bucket = cutoff + 1e-5f;
  if (mode == 1) {
    g.nbins = n_conf;
    g.cell[0] = g.cell[4] = g.cell[8] = 1.f;
    g.inv[0] = g.inv[4] = g.inv[8] = 1.f;
  } else {
    if (pbc) {
      double iv[9];
      cell_inverse(cell, iv);
      for (int k = 0; k < 9; ++k) {
        g.cell[k] = cell[k];
        g.inv[k] = (float)iv[k];
      }
      for (int d = 0; d < 3; ++d) {
        int nd = cell_buckets(iv, d, bucket);
        if (nd < 1) {
          atomicOr(status, ANI_STATUS_CELL_TOO_SMALL);
          nd = 1;
        }
        g.dims[d] = nd;
      }
    } else {
      float mn[3], mx[3];
      for (int d = 0; d < 3; ++d) {
        mn[d] = box_min[d];
        mx[d] = box_max[d];
        if (mn[d] > mx[d]) mn[d] = mx[d] = 0.f;  // no real atoms
        float ext = (mx[d] - mn[d]) + 2e-3f;
        g.origin[d] = mn[d] - 1e-3f;
        g.cell[4 * d] = ext;
        g.inv[4 * d] = 1.0f / ext;
        int nd = (int)floorf(ext / bucket);
        g.dims[d] = nd < 1 ? 1 : nd;
      }
    }
    const int n_sub = mode == 2 ? n_conf : 1;
    cap_dims(g, (max_bins - 1) / n_sub);
    g.nbins = g.dims[0] * g.dims[1] * g.dims[2] * n_sub;
  }
  return g;
}

// Grid mode 3 (a periodic batch with one cell per conformer), executed by ALL threads of one CTA: thread t inverts
// the cells of conformers t, t + blockDim.x, ... (in double, as compute_grid) and writes their rows of the lattice
// table {cell[9], inverse[9]}; the sub-grid dims common to all conformers are, per axis, the minimum over the
// conformers of the buckets their own cell admits, capped like mode 2.  With C equal cells this is the mode 2 grid.
// Thread 0 gets the grid (cell / inv: those of conformer 0).
__device__ void conformer_lattices(int n_conf, int n_per_conf, const float* __restrict__ cells, float cutoff,
                                   int max_bins, float* __restrict__ lattice, int32_t* __restrict__ status,
                                   ani_grid& out) {
  __shared__ int s_dims[3];
  if (threadIdx.x < 3) s_dims[threadIdx.x] = 0x7fffffff;
  __syncthreads();
  const float bucket = cutoff + 1e-5f;
  int nd_min[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff};
  for (int c = threadIdx.x; c < n_conf; c += blockDim.x) {
    const float* cell = cells + 9 * (size_t)c;
    double iv[9];
    cell_inverse(cell, iv);
    float* L = lattice + (size_t)c * ANI_LATTICE_STRIDE;
    for (int k = 0; k < 9; ++k) {
      L[k] = cell[k];
      L[9 + k] = (float)iv[k];
    }
    for (int d = 0; d < 3; ++d) {
      int nd = cell_buckets(iv, d, bucket);
      if (nd < 1) {
        atomicOr(status, ANI_STATUS_CELL_TOO_SMALL);
        nd = 1;
      }
      nd_min[d] = min(nd_min[d], nd);
    }
  }
  for (int d = 0; d < 3; ++d) atomicMin(&s_dims[d], nd_min[d]);
  __syncthreads();
  if (threadIdx.x != 0) return;
  ani_grid g;
  for (int k = 0; k < 9; ++k) {
    g.cell[k] = lattice[k];   // written by this thread above
    g.inv[k] = lattice[9 + k];
  }
  g.origin[0] = g.origin[1] = g.origin[2] = 0.f;
  for (int d = 0; d < 3; ++d) g.dims[d] = s_dims[d];
  g.pbc = 1;
  g.mode = 3;
  g.n_per_conf = n_per_conf;
  g.n_real = 0;
  cap_dims(g, (max_bins - 1) / n_conf);
  g.nbins = g.dims[0] * g.dims[1] * g.dims[2] * n_conf;
  out = g;
}

// the cell (and its inverse) of conformer `conf`: with LAT (grid mode 3) its row of the lattice table, written in
// the same launch by another CTA (hence the L2 loads), else the grid's own
template <bool LAT>
__device__ __forceinline__ void cell_of(const ani_grid& g, const float* __restrict__ lattice, int conf, float (&cl)[9]) {
#pragma unroll
  for (int k = 0; k < 9; ++k) cl[k] = LAT ? __ldcg(lattice + (size_t)conf * ANI_LATTICE_STRIDE + k) : g.cell[k];
}

template <bool LAT>
__device__ __forceinline__ void inv_of(const ani_grid& g, const float* __restrict__ lattice, int conf, float (&inv)[9]) {
#pragma unroll
  for (int k = 0; k < 9; ++k) inv[k] = LAT ? __ldcg(lattice + (size_t)conf * ANI_LATTICE_STRIDE + 9 + k) : g.inv[k];
}

// one CTA: the lattice table and the grid of a mode 3 preparation in the five-launch form
__global__ void k_lattice_setup(int n_conf, int n_per_conf, const float* __restrict__ cells, float cutoff,
                                int max_bins, float* __restrict__ lattice, ani_grid* __restrict__ grid,
                                int32_t* __restrict__ status) {
  ani_grid g;
  conformer_lattices(n_conf, n_per_conf, cells, cutoff, max_bins, lattice, status, g);
  if (threadIdx.x == 0) *grid = g;
}

// ---------------------------------------------------------------------------------------
// grid setup: one block.  mode 0 + pbc: buckets from the perpendicular widths of the cell
// (>= 1 bucket per cutoff, neighbors.py:618-662 uses edge lengths; widths are the safe
// choice for triclinic cells).  mode 0 without pbc: bounding box of the real atoms.
// ---------------------------------------------------------------------------------------
__global__ void k_grid_setup(const float* __restrict__ coords, const int32_t* __restrict__ species,
                             int n, int n_conf, int n_per_conf, const float* __restrict__ cell, int pbc,
                             int mode, float cutoff, int max_bins, ani_grid* __restrict__ grid,
                             int32_t* __restrict__ status) {
  __shared__ float s_min[3][32], s_max[3][32];
  const int tid = threadIdx.x;
  float lo[3] = {1e30f, 1e30f, 1e30f}, hi[3] = {-1e30f, -1e30f, -1e30f};
  if (mode == 0 && !pbc) {
    for (int a = tid; a < n; a += blockDim.x) {
      if (species[a] < 0) continue;
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        float v = coords[3 * a + d];
        lo[d] = fminf(lo[d], v);
        hi[d] = fmaxf(hi[d], v);
      }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      for (int o = 16; o > 0; o >>= 1) {
        lo[d] = fminf(lo[d], __shfl_xor_sync(ANI_FULL_MASK, lo[d], o));
        hi[d] = fmaxf(hi[d], __shfl_xor_sync(ANI_FULL_MASK, hi[d], o));
      }
      if ((tid & 31) == 0) {
        s_min[d][tid >> 5] = lo[d];
        s_max[d][tid >> 5] = hi[d];
      }
    }
  }
  __syncthreads();
  if (tid != 0) return;
  float mn[3], mx[3];
  for (int d = 0; d < 3; ++d) {
    mn[d] = 1e30f;
    mx[d] = -1e30f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) {
      mn[d] = fminf(mn[d], s_min[d][w]);
      mx[d] = fmaxf(mx[d], s_max[d][w]);
    }
  }
  *grid = compute_grid(n_conf, n_per_conf, cell, pbc, mode, cutoff, max_bins, mn, mx, status);
}

// LAT (grid mode 3): wrap with the lattice of the atom's own conformer, from the lattice table
template <bool LAT = false>
__device__ __forceinline__ void wrapped_position(const ani_grid& g, const float* __restrict__ coords, int a,
                                                 float3& pos, int& bin, const float* __restrict__ lattice = nullptr) {
  float x = coords[3 * a], y = coords[3 * a + 1], z = coords[3 * a + 2];
  if (!LAT && g.mode == 1) {
    pos = make_float3(x, y, z);
    bin = a / g.n_per_conf;
    return;
  }
  float cl[9], inv[9];
  cell_of<LAT>(g, lattice, LAT ? a / g.n_per_conf : 0, cl);
  inv_of<LAT>(g, lattice, LAT ? a / g.n_per_conf : 0, inv);
  float rx = x - g.origin[0], ry = y - g.origin[1], rz = z - g.origin[2];
  float f[3];
  f[0] = rx * inv[0] + ry * inv[3] + rz * inv[6];
  f[1] = rx * inv[1] + ry * inv[4] + rz * inv[7];
  f[2] = rx * inv[2] + ry * inv[5] + rz * inv[8];
  int idx[3];
  float k[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    if (g.pbc) {
      k[d] = floorf(f[d]);  // utils.py:249-250 (map_to_central): frac -= floor(frac)
      f[d] -= k[d];
    }
    int i = (int)floorf(f[d] * (float)g.dims[d]);
    idx[d] = min(max(i, 0), g.dims[d] - 1);
  }
  // Subtract whole lattice vectors from the input position instead of rebuilding it from the
  // fractional coordinates: atoms already inside the cell keep their exact float32 position
  // (the reference's frac @ cell round trip costs ~1e-7 * |cell| of absolute accuracy).
  pos.x = x - (k[0] * cl[0] + k[1] * cl[3] + k[2] * cl[6]);
  pos.y = y - (k[0] * cl[1] + k[1] * cl[4] + k[2] * cl[7]);
  pos.z = z - (k[0] * cl[2] + k[1] * cl[5] + k[2] * cl[8]);
  bin = (idx[0] * g.dims[1] + idx[1]) * g.dims[2] + idx[2];
  if (LAT || g.mode == 2) bin += (a / g.n_per_conf) * (g.dims[0] * g.dims[1] * g.dims[2]);  // the conformer's sub-grid
}

// ---------------------------------------------------------------------------------------
// The phases of the preparation, written once.  Every preparation form (the three-call public API, the five-launch
// sequence, the persistent grid, the cluster) is a sequence of these pieces.  Where the forms read an array
// differently (plain loads, L2 loads of data another CTA wrote in the same launch, a CTA's shared-memory copy), the
// caller passes the read as a functor.
// ---------------------------------------------------------------------------------------
constexpr int LAYOUT_CHUNK = 256;   // atoms per chunk of the species histograms and the row assignment

// bucket of atom a and its slot inside the bucket (arrival order, by atomics)
template <bool LAT = false>
__device__ __forceinline__ void assign_bucket(const ani_grid& g, const float* __restrict__ coords,
                                              const int32_t* __restrict__ species, int a, int32_t* __restrict__ bin_of,
                                              int32_t* __restrict__ slot, int32_t* __restrict__ bin_count,
                                              const float* __restrict__ lattice = nullptr) {
  int bin;
  if (species[a] < 0) {
    bin = g.nbins;  // padding atoms: trash bucket, never a neighbour, never a centre
  } else {
    float3 p;
    wrapped_position<LAT>(g, coords, a, p, bin, lattice);
  }
  bin_of[a] = bin;
  slot[a] = atomicAdd(&bin_count[bin], 1);
}

// Record o (0..26) of bucket b's table of neighbouring buckets: r0 = {first atom, end atom, image code, neighbour
// bucket}, r1 = the image shift in the lattice of the bucket's conformer.  Neighbours stay inside the conformer's
// sub-grid; outside a non-periodic box the neighbour does not exist (empty range, bucket 0).  start(k) reads bin_start[k].
template <bool LAT, class Start>
__device__ __forceinline__ void neighbour_record(const ani_grid& g, const float* __restrict__ lattice, int b, int o,
                                                 Start start, float4& r0, float4& r1) {
  int ix, iy, iz;
  const int base = bucket_coords(g, b, ix, iy, iz);
  int j[3] = {ix + o / 9 - 1, iy + (o / 3) % 3 - 1, iz + o % 3 - 1};
  int w[3];
  for (int d = 0; d < 3; ++d) {
    w[d] = 0;
    if (j[d] < 0) {
      w[d] = -1;
      j[d] += g.dims[d];
    } else if (j[d] >= g.dims[d]) {
      w[d] = 1;
      j[d] -= g.dims[d];
    }
  }
  const bool exists = g.pbc || !(w[0] | w[1] | w[2]);
  int lo = 0, hi = 0;
  const int code = (w[0] + 1) * 9 + (w[1] + 1) * 3 + (w[2] + 1);
  const int nbk = exists ? base + (j[0] * g.dims[1] + j[1]) * g.dims[2] + j[2] : 0;
  if (exists) {
    lo = start(nbk);
    hi = start(nbk + 1);
  }
  const float wx = (float)w[0], wy = (float)w[1], wz = (float)w[2];
  float cl[9];
  cell_of<LAT>(g, lattice, LAT ? base / (g.dims[0] * g.dims[1] * g.dims[2]) : 0, cl);
  r0 = make_float4(__int_as_float(lo), __int_as_float(hi), __int_as_float(code), __int_as_float(nbk));
  r1 = make_float4(wx * cl[0] + wy * cl[3] + wz * cl[6], wx * cl[1] + wy * cl[4] + wz * cl[7],
                   wx * cl[2] + wy * cl[5] + wz * cl[8], 0.f);
}

// Exclusive scan of the bucket counts by one block of WARPS warps (the whole block calls it): store(i, start) for
// i < m, where load(i) reads count i.  Returns the total to every thread.
template <int WARPS, class Load, class Store>
__device__ __forceinline__ int scan_bucket_counts(int m, Load load, Store store) {
  __shared__ int s_warp[WARPS];
  __shared__ int s_carry;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < m; base += blockDim.x) {
    const int i = base + tid;
    const int v = (i < m) ? load(i) : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(ANI_FULL_MASK, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[w] = x;
    __syncthreads();
    if (w == 0) {
      int t = (lane < WARPS) ? s_warp[lane] : 0;
#pragma unroll
      for (int o = 1; o < WARPS; o <<= 1) {
        const int y = __shfl_up_sync(ANI_FULL_MASK, t, o);
        if (lane >= o) t += y;
      }
      if (lane < WARPS) s_warp[lane] = t;  // inclusive over warps
    }
    __syncthreads();
    const int incl = x + ((w == 0) ? 0 : s_warp[w - 1]) + s_carry;
    if (i < m) store(i, incl - v);
    __syncthreads();
    if (tid == blockDim.x - 1) s_carry = incl;
    __syncthreads();
  }
  return s_carry;
}

// The atomics above give an arbitrary order inside a bucket; rank by (species, input index) to make the sorted order
// (and with it every later summation order) deterministic and every bucket species-sorted, as the AEV kernels require.
// The rank of real atom a (species spa) among the bucket's members member(lo .. hi - 1).
template <class Member>
__device__ __forceinline__ int species_index_rank(const int32_t* __restrict__ species, int lo, int hi, int a, int spa,
                                                  Member member) {
  int rank = 0;
  for (int e = lo; e < hi; ++e) {
    const int t = member(e);
    const int spt = species[t];
    rank += (spt < spa) || (spt == spa && t < a);
  }
  return rank;
}

// Atom a (species sp) of bucket b at sorted position i: the sorted arrays, and with a chunk histogram the count of
// a real atom in its 256-atom chunk of the owned sorted slice [lo, hi_real)
template <bool LAT = false>
__device__ __forceinline__ void place_atom(const ani_grid& g, const float* __restrict__ coords,
                                           const float* __restrict__ lattice, int a, int sp, int b, int i,
                                           int32_t* __restrict__ sorted_orig, int32_t* __restrict__ orig_to_sorted,
                                           int32_t* __restrict__ sbin, float4* __restrict__ spos,
                                           int32_t* __restrict__ chunk_hist = nullptr, int lo = 0, int hi_real = 0) {
  sorted_orig[i] = a;
  orig_to_sorted[a] = i;
  sbin[i] = b;
  float3 p = make_float3(0.f, 0.f, 0.f);
  if (sp >= 0) {
    int bb;
    wrapped_position<LAT>(g, coords, a, p, bb, lattice);
  }
  spos[i] = make_float4(p.x, p.y, p.z, __int_as_float(sp));
  if (chunk_hist && sp >= 0 && i >= lo && i < hi_real)
    atomicAdd(&chunk_hist[((i - lo) / LAYOUT_CHUNK) * ANI_MAX_SPECIES + sp], 1);
}

__global__ void k_bin_assign(const float* __restrict__ coords, const int32_t* __restrict__ species, int n,
                             const ani_grid* __restrict__ grid, int32_t* __restrict__ bin_of,
                             int32_t* __restrict__ slot, int32_t* __restrict__ bin_count) {
  int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n) return;
  const ani_grid g = *grid;
  assign_bucket(g, coords, species, a, bin_of, slot, bin_count);
}

// exclusive scan of cnt[0..m-1] -> start[0..m] by one block of 1024 threads (m = nbins + 1, read from grid)
__global__ void k_bin_scan(const int32_t* __restrict__ cnt, ani_grid* grid, int32_t* __restrict__ start) {
  const int m = grid->nbins + 1;
  const int total = scan_bucket_counts<32>(m, [&](int i) { return cnt[i]; }, [&](int i, int v) { start[i] = v; });
  if (threadIdx.x == 0) {
    start[m] = total;
    grid->n_real = start[m - 1];  // everything before the trash bucket
  }
}

__global__ void k_bin_scatter(int n, const int32_t* __restrict__ bin_of, const int32_t* __restrict__ slot,
                              const int32_t* __restrict__ bin_start, int32_t* __restrict__ tmp_list) {
  int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n) return;
  tmp_list[bin_start[bin_of[a]] + slot[a]] = a;
}

__global__ void k_bin_finalize(const float* __restrict__ coords, const int32_t* __restrict__ species, int n,
                               const ani_grid* __restrict__ grid, const int32_t* __restrict__ bin_of,
                               const int32_t* __restrict__ bin_start, const int32_t* __restrict__ tmp_list,
                               int32_t* __restrict__ sorted_orig, int32_t* __restrict__ orig_to_sorted,
                               float4* __restrict__ spos, int32_t* __restrict__ sbin) {
  int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n) return;
  const ani_grid g = *grid;
  int b = bin_of[a];
  int lo = bin_start[b], hi = bin_start[b + 1];
  const int spa = species[a];
  int rank = 0;
  if (spa < 0) {
    // trash bucket (padding atoms of a conformer batch, possibly thousands): all of one "species", so the rank is
    // the number of smaller indices -- independent loads, no dependent species gather per entry
    for (int e = lo; e < hi; ++e) rank += tmp_list[e] < a;
  } else {
    rank = species_index_rank(species, lo, hi, a, spa, [&](int e) { return tmp_list[e]; });
  }
  place_atom(g, coords, nullptr, a, spa, b, lo + rank, sorted_orig, orig_to_sorted, sbin, spos);
}

// Per-bucket table of the 27 neighbouring buckets (neighbour_record, with .w = 0 in this form).  The AEV kernel then
// reads 27 records instead of redoing the index wrapping and shift arithmetic for every central atom.
__global__ void k_bucket_ranges(const ani_grid* __restrict__ grid, const int32_t* __restrict__ bin_start,
                                float4* __restrict__ ranges) {
  const ani_grid g = *grid;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = idx / 27, o = idx % 27;
  if (b >= g.nbins || g.mode == 1) return;
  float4 r0, r1;
  neighbour_record<false>(g, nullptr, b, o, [&](int k) { return bin_start[k]; }, r0, r1);
  r0.w = 0.f;
  ranges[2 * (size_t)idx] = r0;
  ranges[2 * (size_t)idx + 1] = r1;
}

// ---------------------------------------------------------------------------------------
// species-grouped row layout (three kernels, deterministic):
//   1. per-chunk species histogram of the owned sorted atoms
//   2. one block: scan chunks per species, pad each species block to ANI_TILE_ROWS rows,
//      emit the tile table
//   3. per-chunk: assign rows (ballot ranks inside the chunk)
// ---------------------------------------------------------------------------------------

// Exclusive scan over the chunks of chunk_hist[c][s], per species, in place (the whole block calls it): s_tot[s] =
// the total of species s.  The histogram is staged through shared memory in slabs so that the serial scan does not
// pay a global-memory round trip per chunk; load(k) reads chunk_hist[k].
template <class Load>
__device__ __forceinline__ void scan_chunk_hist(int n_chunks, int S, int32_t* __restrict__ chunk_hist, Load load,
                                                int* s_tot) {
  __shared__ int s_slab[128 * ANI_MAX_SPECIES];
  const int tid = threadIdx.x;
  int run = 0;
  for (int c0 = 0; c0 < n_chunks; c0 += 128) {
    const int nc = min(128, n_chunks - c0);
    for (int k = tid; k < nc * ANI_MAX_SPECIES; k += blockDim.x) s_slab[k] = load(c0 * ANI_MAX_SPECIES + k);
    __syncthreads();
    if (tid < S) {
      for (int c = 0; c < nc; ++c) {
        const int v = s_slab[c * ANI_MAX_SPECIES + tid];
        s_slab[c * ANI_MAX_SPECIES + tid] = run;
        run += v;
      }
    }
    __syncthreads();
    for (int k = tid; k < nc * ANI_MAX_SPECIES; k += blockDim.x) chunk_hist[c0 * ANI_MAX_SPECIES + k] = s_slab[k];
    __syncthreads();
  }
  if (tid < S) s_tot[tid] = run;
  __syncthreads();
}

// From the species totals s_tot: the first row s_base[s] of every species, each species block padded to whole row
// tiles (s_base[S] = all rows), and the tables that are given (the whole block calls it):
//   species_base[s] = s_base[s];
//   layout_info = {row tiles, rows, owned atoms, 0, [4 + s] first row tile of species s, [4 + S..] total row tiles};
//   tile_species[t] = species of row tile t, -1 for tiles of padding rows only and beyond the layout.
__device__ __forceinline__ void species_rows(int S, int rows_cap, const int* s_tot, int* s_base,
                                             int32_t* __restrict__ species_base, int32_t* __restrict__ layout_info,
                                             int32_t* __restrict__ tile_species) {
  if (threadIdx.x == 0) {
    int row = 0, owned = 0;
    for (int s = 0; s < S; ++s) {
      s_base[s] = row;
      if (species_base) species_base[s] = row;
      owned += s_tot[s];
      row += (s_tot[s] + ANI_TILE_ROWS - 1) / ANI_TILE_ROWS * ANI_TILE_ROWS;
    }
    s_base[S] = row;
    if (layout_info) {
      layout_info[0] = row / ANI_TILE_ROWS;
      layout_info[1] = row;
      layout_info[2] = owned;
      layout_info[3] = 0;
      for (int s = 0; s <= ANI_MAX_SPECIES; ++s) layout_info[4 + s] = (s <= S ? s_base[s] : row) / ANI_TILE_ROWS;
    }
  }
  __syncthreads();
  if (!tile_species) return;
  const int n_tiles_cap = rows_cap / ANI_TILE_ROWS;
  for (int t = threadIdx.x; t < n_tiles_cap; t += blockDim.x) {
    const int r = t * ANI_TILE_ROWS;
    int sp = -1;
    for (int s = 0; s < S; ++s)
      if (r >= s_base[s] && r < s_base[s + 1] && r < s_base[s] + s_tot[s]) sp = s;
    tile_species[t] = sp;
  }
}

// Rows of one 256-atom chunk of the owned sorted slice, whose thread k holds sorted atom i of species sp (-1: none):
// row0(sp) is the first row of the chunk's atoms of species sp, ballots rank the atoms of a species inside the chunk.
// The whole block calls it, with one or more chunks of 8 warps each; s_wcnt holds one row per warp of the block.
template <class Row0>
__device__ __forceinline__ void assign_chunk_rows(int i, int sp, int S, int (*s_wcnt)[ANI_MAX_SPECIES], Row0 row0,
                                                  int32_t* __restrict__ row_of, int32_t* __restrict__ row_atom) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int my_rank = 0;
  for (int s = 0; s < S; ++s) {
    const unsigned m = __ballot_sync(ANI_FULL_MASK, sp == s);
    if (sp == s) my_rank = __popc(m & ((1u << lane) - 1u));
    if (lane == 0) s_wcnt[w][s] = __popc(m);
  }
  __syncthreads();
  if (sp >= 0) {
    int off = 0;
    for (int ww = w - w % (LAYOUT_CHUNK / 32); ww < w; ++ww) off += s_wcnt[ww][sp];   // from the chunk's first warp
    const int row = row0(sp) + off + my_rank;
    row_of[i] = row;
    row_atom[row] = i;
  }
}

__global__ void k_layout_count(const float4* __restrict__ spos, const ani_grid* __restrict__ grid, int lo,
                               int hi, int S, int32_t* __restrict__ chunk_hist) {
  __shared__ int s_h[ANI_MAX_SPECIES];
  const int n_real = grid->n_real;
  hi = min(hi, n_real);
  if (threadIdx.x < ANI_MAX_SPECIES) s_h[threadIdx.x] = 0;
  __syncthreads();
  int i = lo + blockIdx.x * LAYOUT_CHUNK + threadIdx.x;
  int sp = (i < hi) ? __float_as_int(spos[i].w) : -1;
  for (int s = 0; s < S; ++s) {
    unsigned m = __ballot_sync(ANI_FULL_MASK, sp == s);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(&s_h[s], __popc(m));
  }
  __syncthreads();
  if (threadIdx.x < ANI_MAX_SPECIES) chunk_hist[blockIdx.x * ANI_MAX_SPECIES + threadIdx.x] = s_h[threadIdx.x];
}

__global__ void k_layout_scan(int n_chunks, int S, int rows_cap, int32_t* __restrict__ chunk_hist,
                              int32_t* __restrict__ species_base, int32_t* __restrict__ tile_species,
                              int32_t* __restrict__ row_atom, int32_t* __restrict__ layout_info) {
  // chunk_hist[c][s] -> exclusive prefix over chunks (in place); species_base[s] = first row
  __shared__ int s_tot[ANI_MAX_SPECIES];
  __shared__ int s_base[ANI_MAX_SPECIES + 1];
  scan_chunk_hist(n_chunks, S, chunk_hist, [&](int k) { return chunk_hist[k]; }, s_tot);
  species_rows(S, rows_cap, s_tot, s_base, species_base, layout_info, tile_species);
  for (int r = threadIdx.x; r < rows_cap; r += blockDim.x) row_atom[r] = -1;
}

__global__ void k_layout_assign(const float4* __restrict__ spos, const ani_grid* __restrict__ grid, int lo,
                                int hi, int S, const int32_t* __restrict__ chunk_hist,
                                const int32_t* __restrict__ species_base, int32_t* __restrict__ row_of,
                                int32_t* __restrict__ row_atom) {
  __shared__ int s_wcnt[LAYOUT_CHUNK / 32][ANI_MAX_SPECIES];
  const int n_real = grid->n_real;
  hi = min(hi, n_real);
  int i = lo + blockIdx.x * LAYOUT_CHUNK + threadIdx.x;
  int sp = (i < hi) ? __float_as_int(spos[i].w) : -1;
  assign_chunk_rows(i, sp, S, s_wcnt,
                    [&](int s) { return species_base[s] + chunk_hist[blockIdx.x * ANI_MAX_SPECIES + s]; }, row_of,
                    row_atom);
}

// ---------------------------------------------------------------------------------------
// Active 32-column blocks of the AEV: a column belongs to one neighbour species (radial) or one
// species pair (angular); if that species / pair does not occur among the real atoms, the column
// is identically zero for every atom and its gradient is never consumed.
// ---------------------------------------------------------------------------------------
// Is internal column c of the AEV operand live for the element mask?  Internal order (ani_aev_params::ang_pad): radial
// block [0, RL), `pad` never-written columns, angular block of angular_sub columns per element pair.
__device__ __forceinline__ bool aev_column_live(int c, unsigned mask, int S, int n_shf_r, int angular_sub, int out_dim,
                                                int pad) {
  const int RL = S * n_shf_r;
  if (c < RL) return (mask >> (c / n_shf_r)) & 1u;
  c -= pad;
  if (c < RL || c >= out_dim) return false;
  // invert the row-major upper-triangle pair index
  int s1 = 0, rem = (c - RL) / angular_sub;
  while (rem >= S - s1) {
    rem -= S - s1;
    ++s1;
  }
  return ((mask >> s1) & 1u) && ((mask >> (s1 + rem)) & 1u);
}

// Is any column of 32-column block b live?  One thread walks the block: radial columns one by one, angular columns
// pair block by pair block.
__device__ __forceinline__ bool aev_block_live(int b, unsigned mask, int S, int n_shf_r, int angular_sub, int out_dim,
                                               int pad) {
  bool active = false;
  for (int c = b * 32; c < b * 32 + 32 && !active; ++c) active = aev_column_live(c, mask, S, n_shf_r, angular_sub, out_dim, pad);
  return active;
}

// One warp (the whole warp calls it) compacts the live blocks among the nblk blocks (live(b)) into blocks[1 ..], their
// count into blocks[0], and behind the list the element-presence mask and a "changed since the previous call" flag,
// read by the AEV kernel: dead element pairs are skipped, but zero-filled once whenever the composition changes.
template <class Live>
__device__ __forceinline__ void compact_live_blocks(int nblk, unsigned mask, int32_t* __restrict__ blocks, Live live) {
  const int lane = threadIdx.x & 31;
  int count = 0;
  for (int b0 = 0; b0 < nblk; b0 += 32) {
    const int b = b0 + lane;
    const bool active = b < nblk && live(b);
    const unsigned m = __ballot_sync(ANI_FULL_MASK, active);
    if (active) blocks[1 + count + __popc(m & ((1u << lane) - 1u))] = b;
    count += __popc(m);
  }
  if (lane == 0) {
    blocks[0] = count;
    blocks[nblk + 2] = (blocks[nblk + 1] != (int)mask);
    blocks[nblk + 1] = (int)mask;
  }
}

__global__ void k_species_present(const float4* __restrict__ spos, const ani_grid* __restrict__ grid, int n,
                                  int32_t* __restrict__ present) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int sp = (i < n && i < grid->n_real) ? __float_as_int(spos[i].w) : -1;
  unsigned mask = 0;
  for (int s = 0; s < ANI_MAX_SPECIES; ++s)
    if (__any_sync(ANI_FULL_MASK, sp == s)) mask |= 1u << s;
  if ((threadIdx.x & 31) == 0 && mask) atomicOr(present, (int)mask);
}

__global__ void k_active_blocks(const int32_t* __restrict__ present, int S, int n_shf_r, int angular_sub,
                                int out_dim, int ldx, int ang_pad, int32_t* __restrict__ blocks) {
  // one warp; lane b tests the 32 columns of block b (32 blocks per round), a ballot compacts
  const unsigned mask = (unsigned)*present;
  compact_live_blocks(ldx / 32, mask, blocks,
                      [&](int b) { return aev_block_live(b, mask, S, n_shf_r, angular_sub, out_dim, ang_pad); });
}


// ---------------------------------------------------------------------------------------
// Fused per-step preparation (ani_b200_prepare_step): the same work as build_cells +
// species_layout + active_aev_blocks in five launches instead of twelve --
//   P1 grid (inline) + bucket assignment, the last block to finish scans the bucket counts
//   P2 scatter into buckets  +  per-bucket neighbour-range table
//   P3 deterministic (species, input index) order inside buckets, sorted arrays, per-chunk species histogram, element
//      presence mask, zero-fill of the force accumulator
//   P4 (one block) chunk scan, species row bases, tile table, live AEV column blocks
//   P5 row assignment
// Every launch boundary is a grid-wide dependency; nothing is synchronised with the host.
// ---------------------------------------------------------------------------------------
struct PrepArgs {
  const float* coords;
  const int32_t* species;
  int n, n_conf, n_per_conf;
  const float* cell;
  int pbc, mode;
  float cutoff;
  int max_bins;
  ani_grid* grid;
  int32_t *bin_start, *sorted_orig, *orig_to_sorted;
  float4* spos;
  int32_t* sbin;
  float4* ranges;
  int lo, hi, S, rows_cap;
  int32_t *row_of, *row_atom, *tile_species, *layout_info;
  int n_shf_r, angular_sub, out_dim, ldx, ang_pad;
  int32_t* blocks;
  int32_t *bin_of, *slot, *tmp_list, *bin_count, *counter, *present, *chunk_hist, *species_base;
  int n_chunks, inline_setup;
  float* zero_f32;
  int zero_f32_count;
  double* zero_f64;
  int zero_f64_count;
  int32_t* status;
  int32_t* bss;  // [nbins][8] or nullptr: offset inside bucket b of its first atom of species >= s (buckets are species-sorted)
  unsigned long long* trace;  // timing experiments (ANI_B200_PREP_TRACE=1): %globaltimer at the phase boundaries of k_prep_cluster
  float* lattice;  // grid mode 3: [n_conf][ANI_LATTICE_STRIDE] {cell, inverse} per conformer (written by the preparation)
};

// per-bucket species offsets: bss[b][s] = atoms of bucket b with species < s (s = 0..7; bss[b][0] = 0).  With the
// species-sorted order inside a bucket this is where species s starts; the AEV forward kernel reads 27 such rows
// instead of counting the species of ~370 candidates per CTA
__device__ __forceinline__ void bucket_species_offsets(const PrepArgs& A, int b) {
  const int lo = __ldcg(&A.bin_start[b]), hi = __ldcg(&A.bin_start[b + 1]);
  int cnt[ANI_MAX_SPECIES];
#pragma unroll
  for (int k = 0; k < ANI_MAX_SPECIES; ++k) cnt[k] = 0;
  for (int e = lo; e < hi; ++e) {
    const int sp = A.species[__ldcg(&A.tmp_list[e])];
#pragma unroll
    for (int k = 0; k < ANI_MAX_SPECIES; ++k) cnt[k] += (sp == k);
  }
  int run = 0, off[ANI_MAX_SPECIES];
#pragma unroll
  for (int k = 0; k < ANI_MAX_SPECIES; ++k) {
    off[k] = run;
    run += cnt[k];
  }
  int4* dst = reinterpret_cast<int4*>(A.bss + (size_t)b * ANI_MAX_SPECIES);
  dst[0] = make_int4(off[0], off[1], off[2], off[3]);
  dst[1] = make_int4(off[4], off[5], off[6], off[7]);
}

// LAT: grid mode 3 (the grid and the lattice table come from k_lattice_setup, A.inline_setup == 0)
template <bool LAT = false>
__global__ void __launch_bounds__(256) k_prep_assign(const __grid_constant__ PrepArgs A) {
  __shared__ ani_grid sg;
  __shared__ bool s_last;
  const int tid = threadIdx.x;
  if (tid == 0) {
    if (A.inline_setup) {
      const float none[3] = {0.f, 0.f, 0.f};
      sg = compute_grid(A.n_conf, A.n_per_conf, A.cell, A.pbc, A.mode, A.cutoff, A.max_bins, none, none, A.status);
      if (blockIdx.x == 0) *A.grid = sg;
    } else {
      sg = *A.grid;  // written by k_grid_setup (bounding box of an open system)
    }
  }
  __syncthreads();
  const int a = blockIdx.x * blockDim.x + tid;
  if (a < A.n) assign_bucket<LAT>(sg, A.coords, A.species, a, A.bin_of, A.slot, A.bin_count, A.lattice);
  // the last block to get here scans the bucket counts (exclusive) -> bin_start
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(A.counter, 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int m = sg.nbins + 1;
  const int total = scan_bucket_counts<8>(m, [&](int i) { return __ldcg(&A.bin_count[i]); },
                                          [&](int i, int v) { A.bin_start[i] = v; });
  if (tid == 0) {
    A.bin_start[m] = total;
    A.grid->n_real = total - __ldcg(&A.bin_count[m - 1]);  // everything before the trash bucket
  }
}

template <bool LAT = false>
__global__ void __launch_bounds__(256) k_prep_scatter(const __grid_constant__ PrepArgs A) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < A.n) A.tmp_list[A.bin_start[A.bin_of[idx]] + A.slot[idx]] = idx;
  // per-bucket table of the 27 neighbouring buckets (see k_bucket_ranges)
  if (!A.ranges) return;
  const ani_grid g = *A.grid;
  const int b = idx / 27, o = idx % 27;
  if (b >= g.nbins || g.mode == 1) return;
  neighbour_record<LAT>(g, A.lattice, b, o, [&](int k) { return A.bin_start[k]; }, A.ranges[2 * (size_t)idx],
                        A.ranges[2 * (size_t)idx + 1]);
}

template <bool LAT = false>
__global__ void __launch_bounds__(256) k_prep_finalize(const __grid_constant__ PrepArgs A) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  const ani_grid g = *A.grid;
  int sp = -1;
  if (a < A.n) {
    const int b = A.bin_of[a];
    const int lo = A.bin_start[b], hi = A.bin_start[b + 1];
    const int spa = A.species[a];
    int rank;
    if (spa < 0) {
      // padding atoms (trash bucket) are never neighbours nor centres: any order will do -- their arrival slot,
      // instead of ranking thousands of padded entries of a conformer batch against each other
      rank = A.slot[a];
    } else {
      rank = species_index_rank(A.species, lo, hi, a, spa, [&](int e) { return A.tmp_list[e]; });
    }
    sp = A.species[a];   // read again: reusing spa here makes ptxas spill the grid fields around the rank loop
    // with the species histogram of the owned slice, per 256-atom chunk of the SORTED order
    place_atom<LAT>(g, A.coords, A.lattice, a, sp, b, lo + rank, A.sorted_orig, A.orig_to_sorted, A.sbin, A.spos,
                    A.chunk_hist, A.lo, min(A.hi, g.n_real));
  }
  unsigned mask = 0;
  for (int s = 0; s < ANI_MAX_SPECIES; ++s)
    if (__any_sync(ANI_FULL_MASK, sp == s)) mask |= 1u << s;
  if ((threadIdx.x & 31) == 0 && mask) atomicOr(A.present, (int)mask);
  if (A.zero_f32)
    for (int k = a; k < A.zero_f32_count; k += gridDim.x * blockDim.x) A.zero_f32[k] = 0.f;
  if (A.bss)
    for (int b = a; b < g.nbins; b += gridDim.x * blockDim.x) bucket_species_offsets(A, b);
}

__global__ void __launch_bounds__(1024) k_prep_layout(const __grid_constant__ PrepArgs A) {
  __shared__ int s_tot[ANI_MAX_SPECIES];
  __shared__ int s_base[ANI_MAX_SPECIES + 1];
  const int tid = threadIdx.x, S = A.S;
  // ---- live AEV column blocks (warp 31; independent of the scan below)
  if (tid >= 992) {
    const unsigned mask = (unsigned)*A.present;
    compact_live_blocks(A.ldx / 32, mask, A.blocks, [&](int b) {
      return aev_block_live(b, mask, S, A.n_shf_r, A.angular_sub, A.out_dim, A.ang_pad);
    });
  }
  // ---- exclusive scan of the chunk histograms per species (in place), row bases, tile table
  scan_chunk_hist(A.n_chunks, S, A.chunk_hist, [&](int k) { return A.chunk_hist[k]; }, s_tot);
  species_rows(S, A.rows_cap, s_tot, s_base, A.species_base, A.layout_info, A.tile_species);
  for (int r = tid; r < A.rows_cap; r += blockDim.x) A.row_atom[r] = -1;
  if (A.zero_f64)
    for (int k = tid; k < A.zero_f64_count; k += blockDim.x) A.zero_f64[k] = 0.0;
}

// ---------------------------------------------------------------------------------------
// The same five phases as ONE launch: a persistent grid (every block resident) that separates the
// phases with a device-wide barrier instead of a launch boundary -- the preparation is pure dependency
// latency (40 blocks of work at 10 k atoms), so five launch boundaries were most of its 35-44 us.
// The barrier is self-resetting (arrival counter + epoch word in the scratch area, zero at allocation):
// the last block to arrive clears the counter and advances the epoch, the others spin on the epoch.  A
// bounded spin raises ANI_STATUS_INTERNAL instead of hanging the GPU if the state is ever corrupted.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void grid_barrier(int32_t* bar, int32_t* status) {
  __syncthreads();
  if (threadIdx.x == 0) {
    volatile int32_t* epoch = bar + 1;
    const int e = *epoch;
    __threadfence();
    if (atomicAdd(bar, 1) == (int)gridDim.x - 1) {
      bar[0] = 0;
      __threadfence();
      atomicExch(bar + 1, e + 1);
    } else {
      const long long t0 = clock64();
      while (*epoch == e) {
        if (clock64() - t0 > 4000000000LL) {  // ~2 s
          atomicOr(status, ANI_STATUS_INTERNAL);
          break;
        }
      }
    }
    __threadfence();
  }
  __syncthreads();
}

// LAT: grid mode 3 -- block 0 builds the lattice table and the grid in phase 0, the other blocks read the grid after
// the first barrier
template <bool LAT = false>
__global__ void __launch_bounds__(256) k_prep_fused(const __grid_constant__ PrepArgs A, int32_t* bar, int zeroed) {
  __shared__ ani_grid sg;
  __shared__ int s_tot[ANI_MAX_SPECIES];
  __shared__ int s_base[ANI_MAX_SPECIES + 1];
  __shared__ int s_wcnt[LAYOUT_CHUNK / 32][ANI_MAX_SPECIES];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int gstride = gridDim.x * blockDim.x, gtid = blockIdx.x * blockDim.x + tid;
  const int n = A.n, S = A.S;
  // ---- phase 0: the grid (every block computes its own copy) + zero-fill of the counters
  if (LAT) {
    if (blockIdx.x == 0) {
      conformer_lattices(A.n_conf, A.n_per_conf, A.cell, A.cutoff, A.max_bins, A.lattice, A.status, sg);
      if (tid == 0) *A.grid = sg;
    }
  } else if (tid == 0) {
    if (A.inline_setup) {
      const float none[3] = {0.f, 0.f, 0.f};
      sg = compute_grid(A.n_conf, A.n_per_conf, A.cell, A.pbc, A.mode, A.cutoff, A.max_bins, none, none, A.status);
      if (blockIdx.x == 0) *A.grid = sg;
    } else {
      sg = *A.grid;  // written by k_grid_setup (bounding box of an open system)
    }
  }
  for (int k = gtid; k < zeroed; k += gstride) A.bin_count[k] = 0;
  grid_barrier(bar, A.status);
  if (LAT && blockIdx.x != 0) {
    if (tid < (int)(sizeof(ani_grid) / 4))
      reinterpret_cast<int*>(&sg)[tid] = __ldcg(reinterpret_cast<const int*>(A.grid) + tid);
    __syncthreads();
  }
  // ---- phase 1: bucket of every atom, slot inside the bucket by atomics
  for (int a = gtid; a < n; a += gstride)
    assign_bucket<LAT>(sg, A.coords, A.species, a, A.bin_of, A.slot, A.bin_count, A.lattice);
  grid_barrier(bar, A.status);
  // ---- phase 1b: block 0 scans the bucket counts (exclusive) -> bin_start, n_real
  if (blockIdx.x == 0) {
    const int m = sg.nbins + 1;
    const int total = scan_bucket_counts<8>(m, [&](int i) { return __ldcg(&A.bin_count[i]); },
                                            [&](int i, int v) { A.bin_start[i] = v; });
    if (tid == 0) {
      A.bin_start[m] = total;
      A.grid->n_real = total - __ldcg(&A.bin_count[m - 1]);  // everything before the trash bucket
    }
  }
  grid_barrier(bar, A.status);
  const int n_real = __ldcg(&A.grid->n_real);
  auto start = [&](int k) { return __ldcg(&A.bin_start[k]); };
  // ---- phase 2: scatter into buckets + per-bucket table of the 27 neighbouring buckets
  {
    const long long t2 = A.ranges ? max((long long)n, (long long)sg.nbins * 27) : (long long)n;
    for (long long idx = gtid; idx < t2; idx += gstride) {
      if (idx < n) A.tmp_list[start(A.bin_of[idx]) + A.slot[idx]] = (int)idx;
      if (!A.ranges || sg.mode == 1) continue;
      const int b = (int)(idx / 27), o = (int)(idx % 27);
      if (b >= sg.nbins) continue;
      neighbour_record<LAT>(sg, A.lattice, b, o, start, A.ranges[2 * (size_t)idx], A.ranges[2 * (size_t)idx + 1]);
    }
  }
  grid_barrier(bar, A.status);
  // ---- phase 3: deterministic (species, input index) order inside buckets, sorted arrays, per-chunk species
  //      histogram, element presence mask, zero-fill of the force accumulator
  {
    const int hi_real = min(A.hi, n_real);
    unsigned mask = 0;
    for (int base = blockIdx.x * blockDim.x; base < n; base += gstride) {  // warp-uniform trip count
      const int a = base + tid;
      int sp = -1;
      if (a < n) {
        const int b = A.bin_of[a];
        const int lo = start(b), hi = start(b + 1);
        sp = A.species[a];
        const int rank = sp < 0 ? A.slot[a]   // padding atoms: arrival order (see k_prep_finalize)
                                : species_index_rank(A.species, lo, hi, a, sp,
                                                     [&](int e) { return __ldcg(&A.tmp_list[e]); });
        place_atom<LAT>(sg, A.coords, A.lattice, a, sp, b, lo + rank, A.sorted_orig, A.orig_to_sorted, A.sbin, A.spos,
                        A.chunk_hist, A.lo, hi_real);
      }
      for (int s = 0; s < ANI_MAX_SPECIES; ++s)
        if (__any_sync(ANI_FULL_MASK, sp == s)) mask |= 1u << s;
    }
    if (lane == 0 && mask) atomicOr(A.present, (int)mask);
    if (A.zero_f32)
      for (int k = gtid; k < A.zero_f32_count; k += gstride) A.zero_f32[k] = 0.f;
    if (A.bss)
      for (int b = gtid; b < sg.nbins; b += gstride) bucket_species_offsets(A, b);
  }
  grid_barrier(bar, A.status);
  // ---- phase 4: block 0: chunk scan, species row bases, tile table, live AEV column blocks;
  //      every block: row_atom = -1
  for (int r = gtid; r < A.rows_cap; r += gstride) A.row_atom[r] = -1;
  if (blockIdx.x == 0) {
    if (w == 7) {
      const unsigned mask = (unsigned)__ldcg(A.present);
      compact_live_blocks(A.ldx / 32, mask, A.blocks, [&](int b) {
        return aev_block_live(b, mask, S, A.n_shf_r, A.angular_sub, A.out_dim, A.ang_pad);
      });
    }
    scan_chunk_hist(A.n_chunks, S, A.chunk_hist, [&](int k) { return __ldcg(&A.chunk_hist[k]); }, s_tot);
    species_rows(S, A.rows_cap, s_tot, s_base, A.species_base, A.layout_info, A.tile_species);
    if (A.zero_f64)
      for (int k = tid; k < A.zero_f64_count; k += blockDim.x) A.zero_f64[k] = 0.0;
  }
  grid_barrier(bar, A.status);
  // ---- phase 5: row assignment, one 256-atom chunk of the owned sorted slice at a time
  {
    const int hi_real = min(A.hi, n_real);
    for (int c = blockIdx.x; c < A.n_chunks; c += gridDim.x) {
      const int i = A.lo + c * LAYOUT_CHUNK + tid;
      const int sp = (i < hi_real) ? __float_as_int(__ldcg(&A.spos[i]).w) : -1;
      assign_chunk_rows(i, sp, S, s_wcnt, [&](int s) {
        return __ldcg(&A.species_base[s]) + __ldcg(&A.chunk_hist[c * ANI_MAX_SPECIES + s]);
      }, A.row_of, A.row_atom);
      __syncthreads();
    }
  }
}

// ---------------------------------------------------------------------------------------
// The preparation as ONE THREAD-BLOCK CLUSTER (k_prep_cluster): at MD sizes (10 k atoms = 40 blocks of
// work) the step above is nothing but dependency latency -- seven device-wide barriers (atomic + spin on
// an L2 word, ~2.5 us each) around phases of one or two dependent global round trips.  Eight CTAs of 1024
// threads on one GPC do the same work with the hardware cluster barrier (barrier.cluster, release /
// acquire at cluster scope) between the phases, and four barriers instead of seven:
//   * every CTA scans the bucket counts into ITS OWN shared-memory copy of bin_start (CTA 0 also
//     writes the global array), so the scan needs no barrier behind it and the scatter / neighbour-range
//     table / ordering phases read bin_start from shared memory;
//   * the (species, input index) order inside a bucket is found by ONE WARP PER BUCKET: the lanes load
//     the bucket's members once (two dependent loads in all) and rank them with shuffles, instead of every
//     atom walking its bucket through global memory (a chain of 2 x bucket-size dependent loads);
//   * every CTA scans the chunk histograms itself (shared memory), so the row assignment follows
//     without another barrier; CTA 0 writes the layout words, the tile table and the live AEV blocks.
// Outputs are bit-identical to k_prep_fused (tests/test_gpu_prepare.py::test_preparation_forms).
// Used for periodic single systems up to PREP_CLUSTER_MAX_ATOMS atoms and PREP_CLUSTER_MAX_BINS buckets;
// larger problems have enough work per phase for the whole device and keep the persistent-grid kernel.
// ---------------------------------------------------------------------------------------
constexpr int PREP_CLUSTER_CTAS = 8;          // portable cluster size; 16 (opt-in) where the device can place it
constexpr int PREP_CLUSTER_THREADS = 1024;
constexpr int PREP_CLUSTER_MAX_ATOMS = 16384;
constexpr int PREP_CLUSTER_MAX_BINS = PREP_CLUSTER_MAX_ATOMS + 1;   // max_bins - 1 = n + 1 buckets at most: the
                                                                    // shared-memory copy of bin_start is dynamic
constexpr int PREP_CLUSTER_MAX_CHUNKS = PREP_CLUSTER_MAX_ATOMS / LAYOUT_CHUNK;
constexpr int MAX_AEV_BLOCKS = 64;   // ldx / 32 (gemm_tc.cuh: MAX_BLOCKS)

__device__ __forceinline__ void prep_cluster_barrier() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

__global__ void __launch_bounds__(PREP_CLUSTER_THREADS, 1)
    k_prep_cluster(const __grid_constant__ PrepArgs A) {
  extern __shared__ int s_start[];   // [nbins + 2]: this CTA's copy of bin_start
  __shared__ ani_grid sg;
  __shared__ int s_live[MAX_AEV_BLOCKS];
  __shared__ int s_hist[PREP_CLUSTER_MAX_CHUNKS * ANI_MAX_SPECIES];   // exclusive scan over the chunks, per species
  __shared__ int s_tot[ANI_MAX_SPECIES];
  __shared__ int s_base[ANI_MAX_SPECIES + 1];
  __shared__ int s_wcnt[PREP_CLUSTER_THREADS / 32][ANI_MAX_SPECIES];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int gstride = gridDim.x * blockDim.x, gtid = blockIdx.x * blockDim.x + tid;
  const int n = A.n, S = A.S;
  auto stamp = [&](int k) {
    if (A.trace && gtid == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      A.trace[k] = t;
    }
  };
  stamp(0);
  // ---- phase 0: the grid (every CTA its own copy) + zero-fill of the counters that are used below
  if (tid == 0) {
    const float none[3] = {0.f, 0.f, 0.f};
    sg = compute_grid(A.n_conf, A.n_per_conf, A.cell, A.pbc, A.mode, A.cutoff, A.max_bins, none, none, A.status);
    if (blockIdx.x == 0) *A.grid = sg;
  }
  __syncthreads();
  stamp(1);
  const int nbins = sg.nbins;
  {
    // bin_count[0 .. nbins] | counter | present | chunk_hist[(n_chunks + 1) * 8] are contiguous, but bin_count is
    // max_bins + 1 long: two ranges
    for (int k = gtid; k <= nbins; k += gstride) A.bin_count[k] = 0;
    const int tail = 2 + (A.n_chunks + 1) * ANI_MAX_SPECIES;
    for (int k = gtid; k < tail; k += gstride) A.counter[k] = 0;
  }
  prep_cluster_barrier();
  stamp(2);
  // ---- phase 1: bucket of every atom, slot inside the bucket by atomics
  for (int a = gtid; a < n; a += gstride) assign_bucket(sg, A.coords, A.species, a, A.bin_of, A.slot, A.bin_count);
  // (independent of everything else, in the shadow of the atomics' round trip) the force accumulator, the row table and
  // the conformer energies start from zero / -1; the row table is written again two cluster barriers further down
  if (A.zero_f32)
    for (int k = gtid; k < A.zero_f32_count; k += gstride) A.zero_f32[k] = 0.f;
  for (int r = gtid; r < A.rows_cap; r += gstride) A.row_atom[r] = -1;
  if (A.zero_f64)
    for (int k = gtid; k < A.zero_f64_count; k += gstride) A.zero_f64[k] = 0.0;
  stamp(3);
  prep_cluster_barrier();
  stamp(4);
  // ---- phase 1b: EVERY CTA scans the bucket counts (exclusive) into its shared-memory bin_start
  {
    const int m = nbins + 1;
    const int total = scan_bucket_counts<PREP_CLUSTER_THREADS / 32>(m, [&](int i) { return __ldcg(&A.bin_count[i]); },
                                                                    [&](int i, int v) {
                                                                      s_start[i] = v;
                                                                      if (blockIdx.x == 0) A.bin_start[i] = v;
                                                                    });
    if (tid == 0) {
      s_start[m] = total;
      if (blockIdx.x == 0) {
        A.bin_start[m] = total;
        A.grid->n_real = s_start[nbins];  // everything before the trash bucket
      }
    }
    __syncthreads();
  }
  const int n_real = s_start[nbins];
  stamp(5);
  // ---- phase 2: scatter into buckets + per-bucket table of the 27 neighbouring buckets
  {
    const int t2 = A.ranges ? max(n, nbins * 27) : n;
    for (int idx = gtid; idx < t2; idx += gstride) {
      if (idx < n) A.tmp_list[s_start[A.bin_of[idx]] + A.slot[idx]] = idx;
      if (!A.ranges || sg.mode != 0) continue;
      const int b = idx / 27, o = idx % 27;
      if (b >= nbins) continue;
      neighbour_record<false>(sg, nullptr, b, o, [&](int k) { return s_start[k]; }, A.ranges[2 * (size_t)idx],
                              A.ranges[2 * (size_t)idx + 1]);
    }
  }
  stamp(6);
  prep_cluster_barrier();
  stamp(7);
  // ---- phase 3: one warp per bucket: deterministic (species, input index) order, sorted arrays, per-chunk
  //      species histogram, element presence mask, per-bucket species offsets
  {
    const int hi_real = min(A.hi, n_real);
    const int nwarps = gstride >> 5;
    unsigned present = 0;
    // (the first 32 members of the warp's NEXT bucket are loaded before the current one is ranked: the two dependent
    // loads per bucket overlap the shuffles of the previous one)
    auto load_members = [&](int base, int hi, int& a, int& spa) {
      const int e = base + lane;
      a = e < hi ? __ldcg(&A.tmp_list[e]) : 0x7fffffff;
      spa = e < hi ? A.species[a] : 0x7fff;
    };
    int b = gtid >> 5, pre_a = 0x7fffffff, pre_sp = 0x7fff;
    if (b <= nbins) load_members(s_start[b], s_start[b + 1], pre_a, pre_sp);
    for (; b <= nbins; b += nwarps) {
      const int lo = s_start[b], hi = s_start[b + 1];
      const int first_a = pre_a, first_sp = pre_sp;
      if (b + nwarps <= nbins) load_members(s_start[b + nwarps], s_start[b + nwarps + 1], pre_a, pre_sp);
      int below[ANI_MAX_SPECIES];   // members with species < k (lane-uniform)
#pragma unroll
      for (int k = 0; k < ANI_MAX_SPECIES; ++k) below[k] = 0;
      for (int base = lo; base < hi; base += 32) {
        const int e = base + lane;
        const bool valid = e < hi;
        int a = first_a, spa = first_sp;
        if (base != lo) load_members(base, hi, a, spa);
        int rank = 0;
        if (b == nbins) rank = valid ? A.slot[a] : 0;   // padding atoms: arrival order (see k_prep_finalize)
        for (int base2 = lo; base2 < hi && b < nbins; base2 += 32) {
          int t = a, spt = spa;
          if (base2 != base) {
            const int e2 = base2 + lane;
            t = e2 < hi ? __ldcg(&A.tmp_list[e2]) : 0x7fffffff;
            spt = e2 < hi ? A.species[t] : 0x7fff;
          }
          const int cnt = min(32, hi - base2);
          for (int k = 0; k < cnt; ++k) {
            const int tk = __shfl_sync(ANI_FULL_MASK, t, k), sk = __shfl_sync(ANI_FULL_MASK, spt, k);
            rank += (sk < spa) || (sk == spa && tk < a);
          }
        }
#pragma unroll
        for (int k = 1; k < ANI_MAX_SPECIES; ++k) below[k] += __popc(__ballot_sync(ANI_FULL_MASK, valid && spa < k));
#pragma unroll
        for (int k = 0; k < ANI_MAX_SPECIES; ++k)
          if (__any_sync(ANI_FULL_MASK, valid && spa == k)) present |= 1u << k;
        if (valid)
          place_atom(sg, A.coords, nullptr, a, spa, b, lo + rank, A.sorted_orig, A.orig_to_sorted, A.sbin, A.spos,
                     A.chunk_hist, A.lo, hi_real);
      }
      if (A.bss && b < nbins && lane == 0) {
        int4* dst = reinterpret_cast<int4*>(A.bss + (size_t)b * ANI_MAX_SPECIES);
        dst[0] = make_int4(below[0], below[1], below[2], below[3]);
        dst[1] = make_int4(below[4], below[5], below[6], below[7]);
      }
    }
    if (lane == 0 && present) atomicOr(A.present, (int)present);
  }
  stamp(8);
  prep_cluster_barrier();
  stamp(9);
  // ---- phase 4: EVERY CTA: exclusive scan of the chunk histograms per species (shared memory), species row
  //      bases; CTA 0: layout words, tile table, live AEV column blocks
  {
    const int nc = A.n_chunks;
    if (w < ANI_MAX_SPECIES) {   // warp w scans species w over the chunks
      int run = 0;
      for (int c0 = 0; c0 < nc; c0 += 32) {
        const int c = c0 + lane;
        const int v = c < nc ? __ldcg(&A.chunk_hist[c * ANI_MAX_SPECIES + w]) : 0;
        int x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int y = __shfl_up_sync(ANI_FULL_MASK, x, o);
          if (lane >= o) x += y;
        }
        if (c < nc) s_hist[c * ANI_MAX_SPECIES + w] = run + x - v;
        run += __shfl_sync(ANI_FULL_MASK, x, 31);
      }
      if (lane == 0) s_tot[w] = run;
    }
    __syncthreads();
    const bool cta0 = blockIdx.x == 0;
    species_rows(S, A.rows_cap, s_tot, s_base, nullptr, cta0 ? A.layout_info : nullptr, cta0 ? A.tile_species : nullptr);
    if (cta0) {
      // live 32-column AEV blocks: warp w tests the 32 columns of block w (+32, ...) -- one column per lane -- instead
      // of one lane walking a whole block (the serial walk was 5 us of this kernel's critical path)
      const unsigned mask = (unsigned)__ldcg(A.present);
      const int nblk = A.ldx / 32;
      for (int b = w; b < nblk; b += PREP_CLUSTER_THREADS / 32) {
        const bool active = aev_column_live(b * 32 + lane, mask, S, A.n_shf_r, A.angular_sub, A.out_dim, A.ang_pad);
        const bool live = __any_sync(ANI_FULL_MASK, active);
        if (lane == 0) s_live[b] = live;
      }
      __syncthreads();
      if (w == 0) compact_live_blocks(nblk, mask, A.blocks, [&](int b) { return s_live[b] != 0; });
    }
  }
  stamp(10);
  // ---- phase 5: row assignment, four 256-atom chunks of the owned sorted slice per CTA pass (8 warps each)
  {
    const int hi_real = min(A.hi, n_real);
    constexpr int SUBS = PREP_CLUSTER_THREADS / LAYOUT_CHUNK;   // 4
    for (int c0 = blockIdx.x * SUBS; c0 < A.n_chunks; c0 += gridDim.x * SUBS) {
      const int c = c0 + tid / LAYOUT_CHUNK;
      const int i = A.lo + c * LAYOUT_CHUNK + (tid % LAYOUT_CHUNK);
      const int sp = (c < A.n_chunks && i < hi_real) ? __float_as_int(__ldcg(&A.spos[i]).w) : -1;
      assign_chunk_rows(i, sp, S, s_wcnt, [&](int s) { return s_base[s] + s_hist[c * ANI_MAX_SPECIES + s]; },
                        A.row_of, A.row_atom);
      __syncthreads();
    }
  }
  stamp(11);
}

// ---------------------------------------------------------------------------------------
// Verlet-skin reuse of the bucket grid (neighbors.py:759-884, VerletCellList): a grid built with
// cutoff + skin stays valid -- every pair within the true cutoff is still found in the 27 buckets
// around an atom, and the AEV kernels screen with the true cutoff and the CURRENT positions -- as
// long as no atom has moved more than skin/2 from where it was binned.
//   mode 0 (after a rebuild): remember the binned positions and the lattice vector that wrapped
//          every atom into the cell
//   mode 1 (instead of a rebuild): positions = new coordinates + the remembered lattice vector, in
//          the remembered sorted order; raise `moved` if an atom left its skin/2 sphere
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    k_verlet_positions(int mode, const float* __restrict__ coords, const ani_grid* __restrict__ grid,
                       const int32_t* __restrict__ sorted_orig, int n, float half_skin, float4* __restrict__ spos,
                       float4* __restrict__ ref_pos, float4* __restrict__ ref_shift, int32_t* __restrict__ moved,
                       float* __restrict__ zero_f32, int zero_f32_count, int32_t* __restrict__ changed_flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && i < grid->n_real) {
    const int a = sorted_orig[i];
    const float x = coords[3 * a], y = coords[3 * a + 1], z = coords[3 * a + 2];
    if (mode == 0) {
      const float4 p = spos[i];
      ref_pos[i] = p;
      ref_shift[i] = make_float4(p.x - x, p.y - y, p.z - z, 0.f);
    } else {
      const float4 sh = ref_shift[i], r = ref_pos[i];
      const float px = x + sh.x, py = y + sh.y, pz = z + sh.z;
      const float dx = px - r.x, dy = py - r.y, dz = pz - r.z;
      const float d2 = dx * dx + dy * dy + dz * dz, lim = half_skin * half_skin;
      if (!(d2 <= lim)) atomicOr(moved, 3);             // left the skin/2 sphere (NaN counts as moved)
      else if (d2 > 0.49f * lim) atomicOr(moved, 2);    // beyond 70 % of it: rebuild before the next step
      spos[i] = make_float4(px, py, pz, r.w);
    }
  }
  if (mode == 1) {
    if (zero_f32)
      for (int k = i; k < zero_f32_count; k += gridDim.x * blockDim.x) zero_f32[k] = 0.f;
    // same rows, same composition as the step that built the grid: nothing to zero-fill again
    if (i == 0 && changed_flag) *changed_flag = 0;
  }
}

}  // namespace ani

using namespace ani;

extern "C" int ani_b200_active_aev_blocks(const float* spos, const ani_grid* grid, int n, int num_species,
                                          int n_shf_r, int angular_sub, int out_dim, int ldx, int ang_pad,
                                          int32_t* blocks, int32_t* scratch_i32, void* stream) {
  if (!spos || !grid || !blocks || !scratch_i32) return ANI_ERR_BAD_ARG;
  if (num_species < 1 || num_species > ANI_MAX_SPECIES || n_shf_r < 1 || angular_sub < 1 || ldx % 32 || ang_pad < 0 ||
      out_dim + ang_pad > ldx)
    return ANI_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(scratch_i32, 0, sizeof(int32_t), st);
  k_species_present<<<(n + 255) / 256, 256, 0, st>>>(reinterpret_cast<const float4*>(spos), grid, n, scratch_i32);
  k_active_blocks<<<1, 32, 0, st>>>(scratch_i32, num_species, n_shf_r, angular_sub, out_dim, ldx, ang_pad, blocks);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

// The checks of the grid inputs, common to ani_b200_build_cells and the preparation; n = n_conf * n_per_conf.  Grid
// mode 3 needs the lattice table, which only ani_b200_prepare_step_cells has (lattice == NULL: unsupported).
static int check_grid_args(int n_conf, int n_per_conf, const float* cell, int pbc, int mode, float cutoff, int max_bins,
                           const float* lattice, int& n) {
  if (n_conf < 1 || n_per_conf < 1 || cutoff <= 0.f || max_bins < 2) return ANI_ERR_BAD_ARG;
  if (mode == 0 && n_conf != 1) return ANI_ERR_UNSUPPORTED;
  if (mode == 1 && (pbc || n_conf + 1 > max_bins)) return ANI_ERR_UNSUPPORTED;
  if (mode == 2 && (!pbc || !cell || n_conf + 1 > max_bins)) return ANI_ERR_UNSUPPORTED;
  if (mode == 3 && (!pbc || !cell || !lattice || n_conf + 1 > max_bins)) return ANI_ERR_UNSUPPORTED;
  if (mode < 0 || mode > 3) return ANI_ERR_BAD_ARG;
  if (pbc && !cell) return ANI_ERR_BAD_ARG;
  const long long n_ll = (long long)n_conf * n_per_conf;
  if (n_ll >= (1ll << ANI_IMG_SHIFT)) return ANI_ERR_UNSUPPORTED;
  n = (int)n_ll;
  return ANI_OK;
}

extern "C" int ani_b200_build_cells(const float* coords, const int32_t* species, int n_conf, int n_per_conf,
                                    const float* cell, int pbc, int mode, float cutoff, int max_bins,
                                    ani_grid* grid, int32_t* bin_start, int32_t* sorted_orig,
                                    int32_t* orig_to_sorted, float* spos, int32_t* sbin, float* bucket_ranges,
                                    int32_t* scratch_i32, int32_t* status, void* stream) {
  if (!coords || !species || !grid || !bin_start || !sorted_orig || !orig_to_sorted || !spos || !sbin ||
      !scratch_i32 || !status)
    return ANI_ERR_BAD_ARG;
  int n;
  if (const int err = check_grid_args(n_conf, n_per_conf, cell, pbc, mode, cutoff, max_bins, nullptr, n)) return err;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* bin_of = scratch_i32;
  int32_t* slot = scratch_i32 + n;
  int32_t* tmp_list = scratch_i32 + 2 * (size_t)n;
  int32_t* bin_count = scratch_i32 + 3 * (size_t)n;
  cudaMemsetAsync(bin_count, 0, sizeof(int32_t) * (size_t)(max_bins + 1), st);
  k_grid_setup<<<1, 1024, 0, st>>>(coords, species, n, n_conf, n_per_conf, cell, pbc, mode, cutoff, max_bins,
                                   grid, status);
  const int nb = (n + 255) / 256;
  k_bin_assign<<<nb, 256, 0, st>>>(coords, species, n, grid, bin_of, slot, bin_count);
  k_bin_scan<<<1, 1024, 0, st>>>(bin_count, grid, bin_start);
  k_bin_scatter<<<nb, 256, 0, st>>>(n, bin_of, slot, bin_start, tmp_list);
  k_bin_finalize<<<nb, 256, 0, st>>>(coords, species, n, grid, bin_of, bin_start, tmp_list, sorted_orig,
                                     orig_to_sorted, reinterpret_cast<float4*>(spos), sbin);
  if (bucket_ranges && mode != 1) {
    // nbins is only known on the device: cover the caller's bucket capacity, surplus threads exit
    const long long threads = (long long)(max_bins - 1) * 27;
    k_bucket_ranges<<<(int)((threads + 255) / 256), 256, 0, st>>>(grid, bin_start, reinterpret_cast<float4*>(bucket_ranges));
  }
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_species_layout(const float* spos, const ani_grid* grid, int n, int lo, int hi,
                                       int num_species, int rows_cap, int32_t* row_of, int32_t* row_atom,
                                       int32_t* tile_species, int32_t* layout_info, int32_t* scratch_i32,
                                       void* stream) {
  if (!spos || !grid || !row_of || !row_atom || !tile_species || !layout_info || !scratch_i32)
    return ANI_ERR_BAD_ARG;
  if (num_species < 1 || num_species > ANI_MAX_SPECIES || lo < 0 || hi > n || lo > hi) return ANI_ERR_BAD_ARG;
  if (rows_cap % ANI_TILE_ROWS != 0) return ANI_ERR_BAD_ARG;
  // worst case rows: every species block rounds up by (almost) one tile
  if ((long long)rows_cap < (long long)(hi - lo) + (long long)num_species * (ANI_TILE_ROWS - 1))
    return ANI_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int n_chunks = max(1, (hi - lo + LAYOUT_CHUNK - 1) / LAYOUT_CHUNK);
  int32_t* chunk_hist = scratch_i32;
  int32_t* species_base = scratch_i32 + (size_t)(n_chunks + 1) * ANI_MAX_SPECIES;
  const float4* sp4 = reinterpret_cast<const float4*>(spos);
  k_layout_count<<<n_chunks, LAYOUT_CHUNK, 0, st>>>(sp4, grid, lo, hi, num_species, chunk_hist);
  k_layout_scan<<<1, 1024, 0, st>>>(n_chunks, num_species, rows_cap, chunk_hist, species_base, tile_species,
                                    row_atom, layout_info);
  k_layout_assign<<<n_chunks, LAYOUT_CHUNK, 0, st>>>(sp4, grid, lo, hi, num_species, chunk_hist, species_base,
                                                     row_of, row_atom);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_verlet_positions(int mode, const float* coords, const ani_grid* grid,
                                          const int32_t* sorted_orig, int n, float skin, float* spos, float* ref_pos,
                                          float* ref_shift, int32_t* moved, float* zero_f32, int zero_f32_count,
                                          int32_t* aev_blocks, int ldx, void* stream) {
  if (!coords || !grid || !sorted_orig || !spos || !ref_pos || !ref_shift || !moved || n < 1) return ANI_ERR_BAD_ARG;
  if ((mode != 0 && mode != 1) || !(skin >= 0.f)) return ANI_ERR_BAD_ARG;
  if (zero_f32_count > 0 && !zero_f32) return ANI_ERR_BAD_ARG;
  const int threads = mode == 1 ? max(n, min(zero_f32_count, 1 << 16)) : n;
  k_verlet_positions<<<(threads + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
      mode, coords, grid, sorted_orig, n, 0.5f * skin, reinterpret_cast<float4*>(spos),
      reinterpret_cast<float4*>(ref_pos), reinterpret_cast<float4*>(ref_shift), moved,
      zero_f32_count > 0 ? zero_f32 : nullptr, zero_f32_count, aev_blocks ? aev_blocks + ldx / 32 + 2 : nullptr);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

// ani_b200_prepare_step and ani_b200_prepare_step_cells (lattice: the table of grid mode 3, NULL otherwise)
static int prepare_step(const float* coords, const int32_t* species, int n_conf, int n_per_conf, const float* cell,
                        int pbc, int mode, float cutoff, int max_bins, ani_grid* grid, int32_t* bin_start,
                        int32_t* sorted_orig, int32_t* orig_to_sorted, float* spos, int32_t* sbin, float* bucket_ranges,
                        int lo, int hi, int num_species, int rows_cap, int32_t* row_of, int32_t* row_atom,
                        int32_t* tile_species, int32_t* layout_info, int n_shf_r, int angular_sub, int out_dim, int ldx,
                        int ang_pad, int32_t* aev_blocks, float* zero_f32, int zero_f32_count, double* zero_f64,
                        int zero_f64_count, int32_t* bucket_species, int32_t* scratch_i32, int32_t* status,
                        float* lattice, void* stream) {
  if (!coords || !species || !grid || !bin_start || !sorted_orig || !orig_to_sorted || !spos || !sbin ||
      !row_of || !row_atom || !tile_species || !layout_info || !aev_blocks || !scratch_i32 || !status)
    return ANI_ERR_BAD_ARG;
  int n;
  if (const int err = check_grid_args(n_conf, n_per_conf, cell, pbc, mode, cutoff, max_bins, lattice, n)) return err;
  if (num_species < 1 || num_species > ANI_MAX_SPECIES || lo < 0 || hi > n || lo > hi) return ANI_ERR_BAD_ARG;
  if (rows_cap % ANI_TILE_ROWS != 0) return ANI_ERR_BAD_ARG;
  if ((long long)rows_cap < (long long)(hi - lo) + (long long)num_species * (ANI_TILE_ROWS - 1)) return ANI_ERR_BAD_ARG;
  if (n_shf_r < 1 || angular_sub < 1 || ldx % 32 || ang_pad < 0 || out_dim + ang_pad > ldx) return ANI_ERR_BAD_ARG;
  if ((zero_f32_count > 0 && !zero_f32) || (zero_f64_count > 0 && !zero_f64)) return ANI_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  PrepArgs A;
  A.coords = coords; A.species = species; A.n = n; A.n_conf = n_conf; A.n_per_conf = n_per_conf;
  A.cell = cell; A.pbc = pbc; A.mode = mode; A.cutoff = cutoff; A.max_bins = max_bins;
  A.grid = grid; A.bin_start = bin_start; A.sorted_orig = sorted_orig; A.orig_to_sorted = orig_to_sorted;
  A.spos = reinterpret_cast<float4*>(spos); A.sbin = sbin;
  A.ranges = (bucket_ranges && mode != 1) ? reinterpret_cast<float4*>(bucket_ranges) : nullptr;
  A.lo = lo; A.hi = hi; A.S = num_species; A.rows_cap = rows_cap;
  A.row_of = row_of; A.row_atom = row_atom; A.tile_species = tile_species; A.layout_info = layout_info;
  A.n_shf_r = n_shf_r; A.angular_sub = angular_sub; A.out_dim = out_dim; A.ldx = ldx; A.ang_pad = ang_pad; A.blocks = aev_blocks;
  A.n_chunks = max(1, (hi - lo + LAYOUT_CHUNK - 1) / LAYOUT_CHUNK);
  // scratch: bin_of[n] slot[n] tmp_list[n] | zeroed: bin_count[max_bins+1] counter present chunk_hist | species_base
  A.bin_of = scratch_i32;
  A.slot = scratch_i32 + n;
  A.tmp_list = scratch_i32 + 2 * (size_t)n;
  // (two words at a FIXED place, outside the per-step zero-fill: the state of the device-wide barrier)
  int32_t* grid_bar = scratch_i32 + 3 * (size_t)n;
  A.bin_count = grid_bar + 2;
  A.counter = A.bin_count + max_bins + 1;
  A.present = A.counter + 1;
  A.chunk_hist = A.present + 1;
  A.species_base = A.chunk_hist + (size_t)(A.n_chunks + 1) * ANI_MAX_SPECIES;
  A.zero_f32 = zero_f32_count > 0 ? zero_f32 : nullptr; A.zero_f32_count = zero_f32_count;
  A.zero_f64 = zero_f64_count > 0 ? zero_f64 : nullptr; A.zero_f64_count = zero_f64_count;
  A.status = status;
  A.bss = bucket_species;
  {  // timing experiments: 12 int64 stamps behind species_base, inside the 32 spare ints of the documented scratch
    const char* te = getenv("ANI_B200_PREP_TRACE");
    A.trace = (te && atoi(te) != 0)
                  ? reinterpret_cast<unsigned long long*>((reinterpret_cast<uintptr_t>(A.species_base + ANI_MAX_SPECIES) + 7) & ~(uintptr_t)7)
                  : nullptr;
  }
  A.lattice = lattice;
  const bool lat = mode == 3;
  // (mode 3: the grid comes from k_lattice_setup / block 0 of the persistent grid)
  A.inline_setup = ((mode == 1 || pbc) && !lat) ? 1 : 0;
  const size_t zeroed = (size_t)(max_bins + 1) + 2 + (size_t)(A.n_chunks + 1) * ANI_MAX_SPECIES;
  if (!A.inline_setup && !lat)
    k_grid_setup<<<1, 1024, 0, st>>>(coords, species, n, n_conf, n_per_conf, cell, pbc, mode, cutoff, max_bins,
                                     grid, status);
  const int nb = (n + 255) / 256;
  static int num_sms = 0;
  if (num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
  }
  static const bool fused = []() {
    const char* e = getenv("ANI_B200_PREP_FUSED");  // ANI_B200_PREP_FUSED=0: the five-launch sequence
    return !e || atoi(e) != 0;
  }();
  // periodic single systems of MD size: one thread-block cluster (ANI_B200_PREP_CLUSTER=0: never)
  const char* ce = getenv("ANI_B200_PREP_CLUSTER");
  const bool cluster_ok = (!ce || atoi(ce) != 0) && fused && A.inline_setup && mode == 0 &&
                          n <= PREP_CLUSTER_MAX_ATOMS && max_bins - 1 <= PREP_CLUSTER_MAX_BINS && A.ldx / 32 <= MAX_AEV_BLOCKS;
  if (cluster_ok) {
    // (bin_start copy: nbins + 2 words, nbins <= max_bins - 1 -- NOT bounded by the number of atoms: a dilute system has
    // more buckets than atoms)
    const size_t dyn = sizeof(int32_t) * (size_t)(max_bins + 1);
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(PREP_CLUSTER_THREADS);
    cfg.dynamicSmemBytes = dyn;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.y = attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    // cluster size: 16 CTAs (non-portable, opt-in) if the device can co-schedule them with the largest shared-memory
    // request, else the portable 8; ANI_B200_PREP_CLUSTER_CTAS pins it
    static int cluster_ctas = 0;
    if (cluster_ctas == 0) {
      cudaFuncSetAttribute(k_prep_cluster, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)sizeof(int32_t) * (PREP_CLUSTER_MAX_BINS + 2));
      cluster_ctas = PREP_CLUSTER_CTAS;
      const char* pe = getenv("ANI_B200_PREP_CLUSTER_CTAS");
      const int want = pe ? atoi(pe) : 16;
      if (want == 16 &&
          cudaFuncSetAttribute(k_prep_cluster, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess) {
        cudaLaunchConfig_t probe = cfg;
        probe.gridDim = dim3(16);
        probe.dynamicSmemBytes = sizeof(int32_t) * (PREP_CLUSTER_MAX_BINS + 2);
        attr[0].val.clusterDim.x = 16;
        int nclusters = 0;
        if (cudaOccupancyMaxActiveClusters(&nclusters, k_prep_cluster, &probe) == cudaSuccess && nclusters >= 1)
          cluster_ctas = 16;
      }
      cudaGetLastError();   // a refused probe is not an error of this call
    }
    cfg.gridDim = dim3(cluster_ctas);
    attr[0].val.clusterDim.x = cluster_ctas;
    if (cudaLaunchKernelEx(&cfg, k_prep_cluster, A) != cudaSuccess && cluster_ctas == 16) {
      // the probe said yes but the launch was refused (partitioned device, ...): the portable size from now on
      cudaGetLastError();
      cluster_ctas = PREP_CLUSTER_CTAS;
      cfg.gridDim = dim3(cluster_ctas);
      attr[0].val.clusterDim.x = cluster_ctas;
      cudaLaunchKernelEx(&cfg, k_prep_cluster, A);
    }
  } else if (fused) {
    // one persistent launch, device-wide barriers between the phases; every block must be resident:
    // 2 blocks of 256 threads per SM at most (the kernel allows far more)
    int32_t* bar = grid_bar;
    const int blocks = min(2 * num_sms, max(1, nb));
    if (lat)
      k_prep_fused<true><<<blocks, 256, 0, st>>>(A, bar, (int)zeroed);
    else
      k_prep_fused<<<blocks, 256, 0, st>>>(A, bar, (int)zeroed);
  } else {
    cudaMemsetAsync(A.bin_count, 0, sizeof(int32_t) * zeroed, st);
    const long long t2 = A.ranges ? max((long long)n, (long long)(max_bins - 1) * 27) : (long long)n;
    if (lat) {
      k_lattice_setup<<<1, 256, 0, st>>>(n_conf, n_per_conf, cell, cutoff, max_bins, lattice, grid, status);
      k_prep_assign<true><<<nb, 256, 0, st>>>(A);
      k_prep_scatter<true><<<(int)((t2 + 255) / 256), 256, 0, st>>>(A);
      k_prep_finalize<true><<<nb, 256, 0, st>>>(A);
    } else {
      k_prep_assign<<<nb, 256, 0, st>>>(A);
      k_prep_scatter<<<(int)((t2 + 255) / 256), 256, 0, st>>>(A);
      k_prep_finalize<<<nb, 256, 0, st>>>(A);
    }
    k_prep_layout<<<1, 1024, 0, st>>>(A);
    k_layout_assign<<<A.n_chunks, LAYOUT_CHUNK, 0, st>>>(A.spos, grid, lo, hi, num_species, A.chunk_hist, A.species_base,
                                                        row_of, row_atom);
  }
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_prepare_step(const float* coords, const int32_t* species, int n_conf, int n_per_conf,
                                     const float* cell, int pbc, int mode, float cutoff, int max_bins,
                                     ani_grid* grid, int32_t* bin_start, int32_t* sorted_orig,
                                     int32_t* orig_to_sorted, float* spos, int32_t* sbin, float* bucket_ranges,
                                     int lo, int hi, int num_species, int rows_cap, int32_t* row_of,
                                     int32_t* row_atom, int32_t* tile_species, int32_t* layout_info, int n_shf_r,
                                     int angular_sub, int out_dim, int ldx, int ang_pad, int32_t* aev_blocks,
                                     float* zero_f32,
                                     int zero_f32_count, double* zero_f64, int zero_f64_count,
                                     int32_t* bucket_species, int32_t* scratch_i32, int32_t* status, void* stream) {
  return prepare_step(coords, species, n_conf, n_per_conf, cell, pbc, mode, cutoff, max_bins, grid, bin_start,
                           sorted_orig, orig_to_sorted, spos, sbin, bucket_ranges, lo, hi, num_species, rows_cap, row_of,
                           row_atom, tile_species, layout_info, n_shf_r, angular_sub, out_dim, ldx, ang_pad, aev_blocks,
                           zero_f32, zero_f32_count, zero_f64, zero_f64_count, bucket_species, scratch_i32, status,
                           nullptr, stream);
}

extern "C" int ani_b200_prepare_step_cells(const float* coords, const int32_t* species, int n_conf, int n_per_conf,
                                           const float* cell, int pbc, int mode, float cutoff, int max_bins,
                                           ani_grid* grid, int32_t* bin_start, int32_t* sorted_orig,
                                           int32_t* orig_to_sorted, float* spos, int32_t* sbin, float* bucket_ranges,
                                           int lo, int hi, int num_species, int rows_cap, int32_t* row_of,
                                           int32_t* row_atom, int32_t* tile_species, int32_t* layout_info, int n_shf_r,
                                           int angular_sub, int out_dim, int ldx, int ang_pad, int32_t* aev_blocks,
                                           float* zero_f32, int zero_f32_count, double* zero_f64, int zero_f64_count,
                                           int32_t* bucket_species, int32_t* scratch_i32, int32_t* status,
                                           float* lattice, void* stream) {
  if (!lattice) return ANI_ERR_BAD_ARG;
  if (mode != 3) return ANI_ERR_UNSUPPORTED;
  return prepare_step(coords, species, n_conf, n_per_conf, cell, pbc, mode, cutoff, max_bins, grid, bin_start,
                           sorted_orig, orig_to_sorted, spos, sbin, bucket_ranges, lo, hi, num_species, rows_cap, row_of,
                           row_atom, tile_species, layout_info, n_shf_r, angular_sub, out_dim, ldx, ang_pad, aev_blocks,
                           zero_f32, zero_f32_count, zero_f64, zero_f64_count, bucket_species, scratch_i32, status,
                           lattice, stream);
}
