/*
 * ani_b200.h -- C-ABI of the CUDA-native (H100, sm_90a) ANI energy+force hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  Every entry point takes plain device
 * pointers, sizes and an explicit cudaStream_t (passed as void*), never allocates,
 * never synchronises the host, and returns 0 on success or a negative ANI_ERR_* code
 * (ani_b200_error_string() explains it).  Device-side conditions that the reference
 * reports as exceptions (neighbour overflow, periodic cell smaller than the cutoff)
 * are raised through a device status word that the caller reads when convenient.
 *
 * What each entry point replaces in the reference (paths under /root/reference/torchani):
 *   ani_b200_build_cells        neighbors.py:418-507,554-615 (_cell_list bucketing), utils.py:237-255
 *                               (map_to_central), csrc/cell_list.cpp:266-350
 *   ani_b200_species_layout     nn/_containers.py:412-415 (per-species nonzero/index_select)
 *   ani_b200_active_aev_blocks  (no counterpart: exact block-sparsity of the AEV the reference ignores)
 *   ani_b200_aev_forward        neighbors.py:64-113,968-1002 + aev/_computer.py:274-350;
 *                               csrc/cuaev.cpp:189-246 (cuaev::run / run_with_half_nbrlist),
 *                               csrc/aev.cu:323-472,768-834 (K8/K9), :975-1039 (K4)
 *   ani_b200_aev_backward       csrc/cuaev.cpp:134-163, csrc/aev.cu:474-766,837-967 (K10/K11)
 *   ani_b200_pairs_to_rows, ani_b200_aev_*_rows   aev/_computer.py:251-272, csrc/aev.cu:1128-1208 (K6)
 *   ani_b200_half_neighbor_*    neighbors.py:366-415 (cell_list), :187-212 (all_pairs) -> Neighbors
 *   ani_b200_mlp_forward_backward  nn/_containers.py:377-421,608-651, nn/_core.py:146-167,
 *                               nn/_infer.py:61-216 (BmmEnsemble), csrc/mnp.cpp:63-236 (mnp::run)
 *   ani_b200_mlp_forward / _zero_live_blocks / _mlp_backward   the same, as separate halves
 *   ani_b200_reduce_energies    nn/_containers.py:418-421,633-636, sae.py:54-64
 *   ani_b200_verlet_positions   neighbors.py:759-884 (VerletCellList: reuse of a list built with a skin)
 *   ani_b200_aev_backward(..., virial, ...)   ase.py:164-168 (the "f dot r" virial of the stress)
 *   ani_b200_aev_backward_members  arch.py:403-436 (members_forces: one autograd pass per member)
 *   ani_b200_ensemble_qbc       arch.py:439-485,543-576 (energies_qbcs, force_magnitudes, force_qbc)
 *   ani_b200_pair_potential     potentials/core.py:106-207, potentials/xtb.py:57-77, potentials/zbl.py:68-81
 *                               (RepulsionXTB / RepulsionZBL over the step's own neighbour list); _pairs: over a
 *                               caller-supplied half list, with ghost weights
 *   ani_b200_pair_potential_search  the same and potentials/lj.py, potentials/fixed_coulomb.py (LennardJones,
 *                               RepulsionLJ, DispersionLJ, FixedCoulomb, FixedMNOK) with a neighbour search of their own
 *                               cutoff
 *   ani_b200_dispersion_d3      potentials/dftd3.py:102-311 (TwoBodyDispersionD3, D3(BJ) two-body dispersion with its
 *                               own neighbour search); _pairs: over a caller-supplied half list, with ghost weights
 *   ani_b200_charges            electro.py:29-156 (ChargeNormalizer.forward, DipoleComputer.forward) on the raw outputs of
 *                               a charge network pass (potentials/nnp.py:75-102, SeparateChargesNNPotential)
 *   ani_b200_operand_format     (no counterpart: format of the tensor-core GEMM operands of this build)
 *   ani_b200_md_*               (no counterpart: the reference's MD loop is ASE's VelocityVerlet / Langevin on the host)
 */
#ifndef ANI_B200_H
#define ANI_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ANI_B200_ABI_VERSION 4

#define ANI_MAX_SPECIES 8
#define ANI_MAX_SHFR 32
#define ANI_MAX_SHFA 8
#define ANI_MAX_SHFZ 8
#define ANI_MAX_MEMBERS 16
#define ANI_TILE_ROWS 128 /* rows of the species-grouped AEV matrix per MLP tile */

/* error codes (return values) */
#define ANI_OK 0
#define ANI_ERR_BAD_ARG (-1)
#define ANI_ERR_UNSUPPORTED (-2)
#define ANI_ERR_CUDA (-3)

/* bits of the device status word (int32, written by kernels, never cleared by them) */
#define ANI_STATUS_NBR_OVERFLOW 1   /* an atom has more radial neighbours than nbr_cap   */
#define ANI_STATUS_ANG_OVERFLOW 2   /* an atom has more angular neighbours than ANI_MAX_ANG */
#define ANI_STATUS_CELL_TOO_SMALL 4 /* periodic cell thinner than the cutoff (neighbors.py:402-403) */
#define ANI_STATUS_PAIR_OVERFLOW 8  /* half neighbour list exceeds the caller's capacity */
#define ANI_VIRIAL_SLOTS 64         /* partial virial sums (ani_b200_aev_backward)          */
#define ANI_STATUS_OPERAND_RANGE 16 /* a value left the range of the half-precision GEMM operand pieces */
#define ANI_STATUS_INTERNAL 32      /* a device-side barrier / dependency wait timed out (never expected) */

#define ANI_MAX_ANG 96 /* angular neighbours (<= Rca) one central atom may have */
#define ANI_LATTICE_STRIDE 18 /* floats per conformer of the lattice table of grid mode 3: cell[9], inverse[9] */

/* AEV constants; mirrors the CuaevComputer constructor (csrc/cuaev.cpp:247-278).       */
typedef struct ani_aev_params {
  float rcr, rca;            /* radial / angular cutoffs                                  */
  float eta_r, eta_a, zeta;  /* float32-rounded, as the reference's buffers hold them      */
  int32_t n_shf_r, n_shf_a, n_shf_z;
  int32_t num_species;
  int32_t cutoff_kind;       /* 0 = cosine (cutoffs.py:70-81), 1 = smooth (cutoffs.py:84-101) */
  float shf_r[ANI_MAX_SHFR];
  float shf_a[ANI_MAX_SHFA];
  float cos_z[ANI_MAX_SHFZ]; /* cos / sin of the angular sections ShfZ                     */
  float sin_z[ANI_MAX_SHFZ];
  /* internal column layout of the TILED AEV operand (ani_b200_aev_forward layout 1) and of the dE/dAEV rows the      */
  /* backward kernels read: the angular block starts ang_pad columns after the radial block, so that every element   */
  /* pair's 32 features fill exactly one 32-column GEMM block (ANI-2x: 7 x 16 radial columns + 16 = 128; water then   */
  /* has 5 live blocks instead of 8).  The padding columns are never written (zero) and the packed layer-1 weights    */
  /* hold zeros there.  0 = the reference's column order (always so for plain rows, layout 0).                        */
  int32_t ang_pad;
} ani_aev_params;

/* Device-resident description of the bucket grid, written by ani_b200_build_cells.     */
typedef struct ani_grid {
  float cell[9];   /* rows are lattice vectors (identity-like bounding box without PBC)  */
  float inv[9];    /* inverse: frac = (r - origin) @ inv                                  */
  float origin[3];
  int32_t dims[3]; /* buckets per lattice direction (of one conformer's sub-grid, mode 2)  */
  int32_t pbc;     /* 1 = periodic in all three directions                                */
  int32_t nbins;   /* real buckets (all conformers); padding atoms live in bucket nbins   */
  int32_t mode;    /* 0 = one conformer on a grid, 1 = batch, bucket == conformer,        */
                   /* 2 = periodic batch: one sub-grid of the shared cell per conformer,  */
                   /* 3 = periodic batch, one cell per conformer (cell / inv: conformer 0; */
                   /*     every conformer's lattice is in the lattice table)              */
  int32_t n_per_conf;
  int32_t n_real;  /* number of non-padding atoms (== bin_start[nbins])                  */
} ani_grid;

int ani_b200_abi_version(void);

/* Format of the "tiled operand" matrices this build was compiled for (section 6):             */
/*   parts        16-bit pieces per value: 2 = IEEE half pieces of scale*x, 3 = bfloat16 pieces  */
/*   value_scale  power-of-two scale of AEV / activation operands (1 for bfloat16 pieces)        */
/*   grad_scale   power-of-two scale of gradient operands                                        */
/* No reference counterpart (the reference runs cuBLAS sgemm / TF32 on plain fp32 rows).         */
int ani_b200_operand_format(int32_t* parts, float* value_scale, float* grad_scale);
const char* ani_b200_error_string(int code);
/* Last CUDA error string seen by this library on the calling thread (for ANI_ERR_CUDA). */
const char* ani_b200_last_cuda_error(void);

/* ------------------------------------------------------------------------------------ */
/* 1. Bucket the atoms: wrap into the cell (PBC), assign buckets, stable counting sort.   */
/*    coords  [n_conf*n_per_conf*3] f32, species [n_conf*n_per_conf] i32 (-1 = padding)    */
/*    cell    device f32[9] (rows = lattice vectors) or NULL; pbc 0/1 (all directions)      */
/*    mode 0 requires n_conf == 1; mode 1 requires pbc == 0.                                */
/*    mode 3 (one cell per conformer) is ANI_ERR_UNSUPPORTED here: ani_b200_prepare_step_cells. */
/*    mode 2 (C conformers in one shared periodic cell) requires pbc == 1, a cell and        */
/*    n_conf + 1 <= max_bins, else ANI_ERR_UNSUPPORTED (before any CUDA call).  Buckets are   */
/*    conformer-major: bucket c * nb + local, nb = dims[0]*dims[1]*dims[2], nbins = C * nb;   */
/*    dims come from the cell as in mode 0, capped so that nb <= (max_bins - 1) / n_conf, and  */
/*    neighbour ranges never leave a conformer's sub-grid.  With max_bins = C * (max(64, A+2) */
/*    - 1) + 1 a conformer's sub-grid, wrapped positions and in-bucket order are those of a   */
/*    mode 0 call on that conformer alone (the engine sizes its workspaces so).               */
/*    Outputs (all device):                                                                 */
/*      grid            ani_grid                                                            */
/*      bin_start       i32[max_bins+2]  exclusive scan of bucket populations               */
/*      sorted_orig     i32[n]           bucket-sorted position -> flat input index         */
/*      spos            f32[n*4]         wrapped x,y,z + species (int bits) in sorted order  */
/*      sbin            i32[n]           bucket of each sorted atom                         */
/*      orig_to_sorted  i32[n]           inverse of sorted_orig                             */
/*    Scratch: scratch_i32[3*n + max_bins + 2].                                             */
/*      bucket_ranges   f32[(max_bins-1)*27*8] or NULL: for every bucket the 27 neighbouring  */
/*                      buckets as {first atom, end atom, image code, -} + image shift vector   */
/*                      (modes 0 and 2; lets the AEV kernel skip the index / shift arithmetic)   */
int ani_b200_build_cells(const float* coords, const int32_t* species, int n_conf, int n_per_conf,
                         const float* cell, int pbc, int mode, float cutoff, int max_bins,
                         ani_grid* grid, int32_t* bin_start, int32_t* sorted_orig,
                         int32_t* orig_to_sorted, float* spos, int32_t* sbin, float* bucket_ranges,
                         int32_t* scratch_i32, int32_t* status, void* stream);

/* 2. Species-grouped row layout for the MLP: atoms lo..hi-1 (bucket-sorted positions,     */
/*    clipped to the real atoms) get rows grouped by species, every species block padded    */
/*    to a multiple of ANI_TILE_ROWS.                                                       */
/*      row_of      i32[n]        row of sorted atom i (undefined outside lo..hi-1)         */
/*      row_atom    i32[rows_cap] sorted atom of a row, -1 for padding rows                 */
/*      tile_species i32[rows_cap/ANI_TILE_ROWS]  species of each row tile, -1 = unused      */
/*      layout_info i32[16]: {n_tiles, n_rows, n_owned_atoms, 0, first row tile of species   */
/*                  0..S-1, total row tiles, ...}  (device-side tile lists of the GEMMs)      */
/*    Scratch: scratch_i32[(ceil(n/256)+2) * ANI_MAX_SPECIES + 64].                         */
int ani_b200_species_layout(const float* spos, const ani_grid* grid, int n, int lo, int hi,
                            int num_species, int rows_cap, int32_t* row_of, int32_t* row_atom,
                            int32_t* tile_species, int32_t* layout_info, int32_t* scratch_i32,
                            void* stream);

/* 2b. Active 32-column blocks of the AEV matrix: blocks[0] = count, blocks[1..] = ascending */
/*    block ids whose columns belong to an element / element pair present among the real      */
/*    atoms.  All other AEV columns are identically zero for every atom (and their gradient   */
/*    is never consumed), so the MLP may skip them.  blocks i32[ldx/32 + 3]: the last two words */
/*    hold the element-presence bit mask and a "mask changed since the previous call" flag      */
/*    (together: ani_b200_aev_forward's species_mask); scratch i32[1].                           */
int ani_b200_active_aev_blocks(const float* spos, const ani_grid* grid, int n, int num_species,
                               int n_shf_r, int angular_sub, int out_dim, int ldx, int ang_pad, int32_t* blocks,
                               int32_t* scratch_i32, void* stream);

/* 3. Fused neighbour search + AEV forward for sorted atoms lo..hi-1.                      */
/*      row_of     row of the output matrix for each sorted atom (species-grouped rows for   */
/*                 the fused engine, flat input index for the AEVComputer API)               */
/*      aev        layout 0: f32[rows][ldx], columns 0..out_dim-1 of the atom's row are      */
/*                 overwritten.  layout 1: the "tiled operand" form the MLP consumes          */
/*                 (see below; 6*rows_cap*ldx bytes, rows_cap % 128 == 0, ldx % 32 == 0)      */
/*      nbr_cnt    i32[n]; nbr_list i32[n*nbr_cap]: neighbours within Rcr of every processed  */
/*                 atom as (sorted index | image code << 26); kept for the backward pass      */
/*      bucket_ranges  output of ani_b200_build_cells or NULL (ranges are then derived on the   */
/*                 fly); species_mask: {bit per element present in the system, changed flag} or   */
/*                 NULL: angular blocks of absent element pairs are not rewritten while the       */
/*                 composition is unchanged (they hold zeros from the first call)                 */
/*      bucket_species  output of ani_b200_prepare_step or NULL (needs bucket_ranges): per bucket the offsets of   */
/*                 its species inside the (species-sorted) bucket, i32[nbins][8]; lets the kernel skip the pass that  */
/*                 counts the species of the ~370 staged candidates of a CTA                                          */
int ani_b200_aev_forward(const ani_aev_params* params, const ani_grid* grid,
                         const int32_t* bin_start, const float* spos, const int32_t* sbin,
                         const float* bucket_ranges, const int32_t* bucket_species, const int32_t* species_mask, int n, int lo,
                         int hi, const int32_t* row_of, float* aev, int ldx, int layout,
                         int32_t* nbr_cnt, int32_t* nbr_list, int nbr_cap, int32_t* status,
                         void* stream);

/* 4. AEV backward: grad_aev (same row layout as the forward output) -> dE/dcoords,         */
/*    accumulated (+=, float atomics) into grad_coords f32[n*3] in flat INPUT order.         */
/*    species_mask (as in the forward, or NULL): the gradient blocks of element pairs that   */
/*    do not occur in the system are not read (the block-sparse MLP backward leaves them     */
/*    unwritten).  max_elements (0 = num_species): how many distinct elements the caller      */
/*    expects in the system; it only sizes the kernel's shared-memory gradient table (higher   */
/*    occupancy for few-element systems) -- pairs beyond it are read from global memory, the   */
/*    result never depends on it.  virial (or NULL): f64[ANI_VIRIAL_SLOTS][9], zeroed by the     */
/*    caller; the kernel adds partial sums of W_ab = sum_pairs (dE/dDelta)_a Delta_b, the "f dot r" */
/*    virial of ase.py:164-168 (stress = sum over the slots / volume), row-major a, b.  Grid mode  */
/*    2: f64[n_conf][ANI_VIRIAL_SLOTS][9], the pairs of a central atom go to its conformer's slots. */
int ani_b200_aev_backward(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                          const int32_t* sorted_orig, const int32_t* species_mask, int n, int lo,
                          int hi, const int32_t* row_of, const float* grad_aev, int ldx,
                          const int32_t* nbr_cnt,
                          const int32_t* nbr_list, int nbr_cap, float* grad_coords,
                          int32_t* status, int max_elements, double* virial, void* stream);

/* 3d/4d. The AEV forward and backward of a grid-mode-3 preparation (one cell per conformer,              */
/*    ani_b200_prepare_step_cells): the arguments of ani_b200_aev_forward / _backward plus the lattice      */
/*    table that preparation wrote (device f32[n_conf][ANI_LATTICE_STRIDE], not NULL, else ANI_ERR_BAD_ARG). */
/*    Image shifts are taken in the lattice of the central atom's conformer (its neighbours always lie in  */
/*    that conformer).  A mode-3 grid must only be passed to these two entry points; the virial has the    */
/*    per-conformer layout of mode 2.                                                                       */
int ani_b200_aev_forward_cells(const ani_aev_params* params, const ani_grid* grid,
                               const int32_t* bin_start, const float* spos, const int32_t* sbin,
                               const float* bucket_ranges, const int32_t* bucket_species, const int32_t* species_mask,
                               int n, int lo, int hi, const int32_t* row_of, float* aev, int ldx, int layout,
                               int32_t* nbr_cnt, int32_t* nbr_list, int nbr_cap, int32_t* status,
                               const float* lattice, void* stream);
int ani_b200_aev_backward_cells(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                                const int32_t* sorted_orig, const int32_t* species_mask, int n, int lo,
                                int hi, const int32_t* row_of, const float* grad_aev, int ldx,
                                const int32_t* nbr_cnt, const int32_t* nbr_list, int nbr_cap, float* grad_coords,
                                int32_t* status, int max_elements, double* virial, const float* lattice, void* stream);

/* 4e. AEV backward of EVERY active ensemble member in one launch (members_forces, arch.py:403-436; the force       */
/*    disagreement of query-by-committee active learning).  grad_slabs holds one dE_m/dAEV slab per member m,        */
/*    slab m at grad_slabs + m * slab_stride floats, each in the row layout of ani_b200_aev_backward's grad_aev (the   */
/*    want_backward == 2 output of ani_b200_mlp_step, or ani_b200_mlp_step_resident_members).  members: HOST array    */
/*    of n_members (1..ANI_MAX_MEMBERS) member indices, read at launch; output k (the member order of the caller,     */
/*    e.g. the active order) contracts slab members[k] and is accumulated (+=, float atomics) into                    */
/*    grad_members + k * 3 n, f32[n_members][n][3] in flat INPUT order (zeroed by the caller, e.g. as the zero_f32 of */
/*    the preparation).  Only the columns ani_b200_aev_backward reads are read: the radial block and the angular     */
/*    blocks of element pairs present in species_mask, i.e. the live column blocks the MLP writes.  A warp builds its */
/*    atom's neighbour geometry once and loops over the members, their rows double-buffered in shared memory          */
/*    (shared memory does not depend on n_members).  max_elements as in ani_b200_aev_backward.  No virial, no         */
/*    explicit neighbour rows.  Status: ANI_STATUS_ANG_OVERFLOW as ani_b200_aev_backward.  The _cells form takes the   */
/*    lattice table of grid mode 3 (not NULL).                                                                       */
int ani_b200_aev_backward_members(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                                  const int32_t* sorted_orig, const int32_t* species_mask, int n, int lo, int hi,
                                  const int32_t* row_of, const float* grad_slabs, int ldx, long long slab_stride,
                                  const int32_t* members, int n_members, const int32_t* nbr_cnt,
                                  const int32_t* nbr_list, int nbr_cap, float* grad_members, int32_t* status,
                                  int max_elements, void* stream);
int ani_b200_aev_backward_members_cells(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                                        const int32_t* sorted_orig, const int32_t* species_mask, int n, int lo, int hi,
                                        const int32_t* row_of, const float* grad_slabs, int ldx, long long slab_stride,
                                        const int32_t* members, int n_members, const int32_t* nbr_cnt,
                                        const int32_t* nbr_list, int nbr_cap, float* grad_members, int32_t* status,
                                        int max_elements, const float* lattice, void* stream);

/* 4f. Query-by-committee statistics of an ensemble step (arch.py:439-485, 543-576), from                         */
/*      grad_members     f32[n_members][n][3]  dE_m/dcoords (ani_b200_aev_backward_members), n = n_conf * n_per_conf */
/*      members          HOST i32[n_members]  member index of every output k (as given to the backward)             */
/*      member_atomic    f32[M][n]  the member_atomic_out of ani_b200_reduce_energies (indexed by member index)     */
/*      species          i32[n]  element index, -1 padding;  sae f64[num_species] or NULL                          */
/*    writes (plain stores, nothing accumulated, no zero-fill needed):                                               */
/*      grad             f32[n][3]  mean over the outputs of grad_members (the ensemble's dE/dcoords)               */
/*      atom_stats       f32[3][n]  per atom: mean_k |F_k|, (std_k |F_k| + 1e-8) / (mean + 1e-8) (unbiased std),       */
/*                                  (max_k |F_k| - min_k |F_k| + 1e-8) / (mean + 1e-8); one member: 0 and 1.          */
/*                                  Padding atoms follow the same formulas (their forces are 0)                     */
/*      member_energies  f64[n_members][n_conf]  sum over the conformer's real atoms of member_atomic + sae          */
/*      qbc              f64[n_conf]  std_k(E_k) (unbiased; 0 for one member) / sqrt(real atoms of the conformer)    */
/*    Two launches; raises no status bits.                                                                           */
int ani_b200_ensemble_qbc(const float* grad_members, const int32_t* members, int n_members, const float* member_atomic,
                          const int32_t* species, const double* sae, int n_conf, int n_per_conf, float* grad,
                          float* atom_stats, double* member_energies, double* qbc, void* stream);

/* 4g. Pair potentials over the neighbour list of the step (potentials/core.py:106-207: BasePairPotential;           */
/*    potentials/xtb.py:57-77 RepulsionXTB; potentials/zbl.py:68-81 RepulsionZBL).  With d = max(R, 1e-7) * to_bohr:    */
/*      kind 0 (xTB)  E = a[s][t] / d * exp(-b[s][t] * d^c[s][t])      a = y_ab, b = sqrt_alpha_ab, c = k_rep_ab          */
/*      kind 1 (ZBL)  E = a[s][t] / d * sum_q screen_coeff[q] exp(-screen_exp[q] * b[s][t] * d)                          */
/*                    a = Z_s Z_t, b = (Z_s^p + Z_t^p) / k                                                              */
/*      kind 2 (LennardJones)  E = 4 a[s][t] (x^12 - x^6), x = b[s][t] / d     a = sqrt(eps_s eps_t),                  */
/*      kind 3 (RepulsionLJ)   E = 4 a[s][t] x^12                                  b = (sigma_s + sigma_t) / 2 (A),       */
/*      kind 4 (DispersionLJ)  E = -4 a[s][t] x^6                                  to_bohr = 1: the LJ kinds work in A    */
/*      kind 5 (FixedCoulomb)  E = a[s][t] / d                                 a = q_s q_t / dielectric                 */
/*      kind 6 (FixedMNOK)     E = a[s][t] / sqrt((R to_bohr)^2 + b[s][t]^2)   a = q_s q_t, b = 2 / (eta_s + eta_t);   */
/*                             no clamp of R                                                                          */
/*    times the envelope fc(R; cutoff): cutoff_fn 0 = cosine, 1 = smooth(2, 1e-10), 2 = none (then `cutoff` is not      */
/*    read and no pair is screened out).  Pairs with R > cutoff contribute nothing.  The tables are symmetric.          */
typedef struct ani_pair_params {
  int32_t kind, cutoff_fn, num_species, pad_;
  float cutoff;  /* Angstrom */
  float to_bohr; /* Angstrom -> Bohr */
  float a[ANI_MAX_SPECIES][ANI_MAX_SPECIES];
  float b[ANI_MAX_SPECIES][ANI_MAX_SPECIES];
  float c[ANI_MAX_SPECIES][ANI_MAX_SPECIES];
  float screen_coeff[4], screen_exp[4];
} ani_pair_params;

/*    ani_b200_pair_potential evaluates one potential for the sorted atoms lo..hi-1 over the neighbour words             */
/*    ani_b200_aev_forward left in nbr_cnt / nbr_list (so cutoff <= Rcr of that forward: the list holds nothing beyond)   */
/*    and ADDS, per owned atom i with e_i = 1/2 sum_j E fc (the atomic split of potentials/core.py:196-200):             */
/*      atomic        f32[n]  += e_i                     (flat input order; or NULL)                                    */
/*      energies      f64[n_conf] += sum of e_i           (or NULL)                                                      */
/*      grad_coords   f32[n][3] += dE/dr_i = sum_j d[E fc]/dR (-Delta_ij / R)   (or NULL)                                */
/*      virial        += 1/2 (dE/dDelta_ij)_a (Delta_ij)_b per listed pair, buffers and slot rule of                     */
/*                    ani_b200_aev_backward (or NULL)                                                                   */
/*      member_atomic f32[M][n] row members[k] += e_i and grad_members f32[n_members][n][3] slab k += dE/dr_i for        */
/*                    k < n_members (either may be NULL; members: HOST i32[n_members], read at launch): the reference    */
/*                    adds a pair potential to every ensemble member (arch.py:365-378)                                   */
/*    by plain read-modify-write -- every element has one writer, the atom's owner -- so the call must be ordered on    */
/*    the stream after the kernels that produce those buffers (ani_b200_aev_backward[_members],                          */
/*    ani_b200_reduce_energies) and before their consumers (ani_b200_ensemble_qbc, the all-reduce).  energies and the    */
/*    virial take float64 atomics.  The per-rank results of a sharded run add up to the full answer.  One launch; no     */
/*    status bits.  The _cells form is for grid mode 3 and takes its lattice table (not NULL).                          */
int ani_b200_pair_potential(const ani_pair_params* params, const ani_grid* grid, const float* spos,
                            const int32_t* sorted_orig, int n, int lo, int hi, int n_conf, int n_per_conf,
                            const int32_t* nbr_cnt, const int32_t* nbr_list, int nbr_cap, float* atomic,
                            double* energies, float* grad_coords, double* virial, float* member_atomic,
                            float* grad_members, const int32_t* members, int n_members, void* stream);
int ani_b200_pair_potential_cells(const ani_pair_params* params, const ani_grid* grid, const float* spos,
                                  const int32_t* sorted_orig, int n, int lo, int hi, int n_conf, int n_per_conf,
                                  const int32_t* nbr_cnt, const int32_t* nbr_list, int nbr_cap, float* atomic,
                                  double* energies, float* grad_coords, double* virial, float* member_atomic,
                                  float* grad_members, const int32_t* members, int n_members, const float* lattice,
                                  void* stream);
/*    The same potential over a caller-supplied HALF pair list (the reference's Neighbors tuple: flat input indices,    */
/*    diff_vectors = x[idx0] - x[idx1] + shift): species i32[n_conf * n_per_conf] (-1 padding), ghost_flags u8 per atom  */
/*    or NULL -- a pair that touches a ghost atom counts half (potentials/core.py:170-177).  ADDS (float atomics; any    */
/*    of them may be NULL) atomic f32[n], energies f64[n_conf] and grad_coords f32[n][3] = dE/dcoords.                   */
int ani_b200_pair_potential_pairs(const ani_pair_params* params, const int32_t* species, const int64_t* idx0,
                                  const int64_t* idx1, const float* distances, const float* diff_vectors,
                                  const uint8_t* ghost_flags, int64_t num_pairs, int n_conf, int n_per_conf,
                                  float* atomic, double* energies, float* grad_coords, void* stream);
/*    ani_b200_pair_potential_search evaluates one potential of any kind for the sorted atoms lo..hi-1 over a neighbour  */
/*    search of its own cutoff on the grid of ani_b200_prepare_step (bin_start, spos, sorted_orig of that preparation),  */
/*    the search of ani_b200_dispersion_d3 (4h): per lattice direction ceil((cutoff + skin) / bucket width) buckets, a   */
/*    neighbour inside the cutoff at two images counts twice.  cutoff_fn 2 means no cutoff and is for open systems      */
/*    (grid modes 0 and 1), whose stencil then spans the grid or the conformer's bucket.  Periodic widths must be >=      */
/*    cutoff + skin, else ANI_STATUS_CELL_TOO_SMALL is OR-ed into status and the atoms of that cell write nothing.       */
/*    Outputs, add-only contract, ordering and member rules are those of ani_b200_pair_potential.  One launch.  The      */
/*    _cells form is for grid mode 3 and takes its lattice table (not NULL).                                             */
int ani_b200_pair_potential_search(const ani_pair_params* params, const ani_grid* grid, const int32_t* bin_start,
                                   const float* spos, const int32_t* sorted_orig, int n, int lo, int hi, int n_conf,
                                   int n_per_conf, float skin, float* atomic, double* energies, float* grad_coords,
                                   double* virial, float* member_atomic, float* grad_members, const int32_t* members,
                                   int n_members, int32_t* status, void* stream);
int ani_b200_pair_potential_search_cells(const ani_pair_params* params, const ani_grid* grid,
                                         const int32_t* bin_start, const float* spos, const int32_t* sorted_orig,
                                         int n, int lo, int hi, int n_conf, int n_per_conf, float skin, float* atomic,
                                         double* energies, float* grad_coords, double* virial, float* member_atomic,
                                         float* grad_members, const int32_t* members, int n_members, int32_t* status,
                                         const float* lattice, void* stream);

/* 4h. D3(BJ) two-body dispersion (potentials/dftd3.py:140-311, TwoBodyDispersionD3) with its own neighbour search    */
/*    over the step's bucket grid (its cutoff, 8 A in the reference's models, is beyond Rcr).  With d = R * to_bohr:       */
/*      CN_i  = sum_j 1 / (1 + exp(-k1 (k2 (rcov[s_i] + rcov[s_j]) / d - 1)))     (every pair within the cutoff)          */
/*      C6_ij = (sum_pq C6ref_pq L_pq + 1e-35) / (sum_pq L_pq + 1e-35),  over the pq with C6ref_pq > 0,              */
/*              L_pq = exp(-k3 ((CN_i - CNa_pq)^2 + (CN_j - CNb_pq)^2))  (the largest L is factored out of both sums and */
/*              the 1e-35; no positive C6ref: C6 = 1, dC6/dCN = 0)                                                        */
/*      E_ij  = -(s6 C6 / (d^6 + damp6) + s8 c8_scale C6 / (d^8 + damp8)) fc(R; cutoff)                                  */
/*    damp6/8[s][t] = (a1 R0_st + a2)^6/8 (Bohr^6/8), c8_scale[s][t] = 3 sqrt_charge_st; cutoff_fn as ani_pair_params.   */
/*    a1, a2 are informational (damp6/8 are what the kernels read).  Tables: device f32[S][S][25][4], per element pair   */
/*    (s, t) and reference pair (p, q) = 5 p + q the values {C6ref, CNa, CNb, 0} (precalc_coeff6, precalc_coordnums_a/b). */
typedef struct ani_d3_params {
  int32_t cutoff_fn, num_species;
  float cutoff;  /* Angstrom */
  float to_bohr; /* Angstrom -> Bohr */
  float s6, s8, a1, a2;
  float k1, k2, k3, pad_;
  float rcov[ANI_MAX_SPECIES]; /* Bohr */
  float damp6[ANI_MAX_SPECIES][ANI_MAX_SPECIES];
  float damp8[ANI_MAX_SPECIES][ANI_MAX_SPECIES];
  float c8_scale[ANI_MAX_SPECIES][ANI_MAX_SPECIES];
} ani_d3_params;

/*    ani_b200_dispersion_d3 evaluates the term for the grid of ani_b200_prepare_step (bin_start, spos, sorted_orig of     */
/*    that preparation; cutoff_fn 0 or 1, a finite cutoff).  Per lattice direction the search reaches                     */
/*    ceil((cutoff + skin) / bucket width) buckets; a neighbour inside the cutoff at two images counts twice.  Periodic   */
/*    widths must be >= cutoff + skin, else ANI_STATUS_CELL_TOO_SMALL is OR-ed into status and nothing else is written.   */
/*    Three launches: cn (f32[n], scratch) of every real atom, then dedcn (f32[n], scratch) of every real atom together   */
/*    with the energies / direct gradient / direct virial of the owned atoms lo..hi-1, then (only if grad_coords,         */
/*    grad_members or virial is given) the coordination-number chain of the gradient and virial of the owned atoms.      */
/*    Outputs, add-only contract and member rules are those of ani_b200_pair_potential (4g): plain read-modify-write of    */
/*    atomic, grad_coords, member_atomic, grad_members by the atom's owner; float64 atomics into energies and the virial  */
/*    slots.  The per-rank results of a sharded run add up to the full answer (cn and dedcn are computed on every rank).  */
/*    The _cells form is for grid mode 3 and takes its lattice table (not NULL).                                          */
int ani_b200_dispersion_d3(const ani_d3_params* params, const float* tables, const ani_grid* grid,
                           const int32_t* bin_start, const float* spos, const int32_t* sorted_orig, int n, int lo,
                           int hi, int n_conf, int n_per_conf, float skin, float* cn, float* dedcn, float* atomic,
                           double* energies, float* grad_coords, double* virial, float* member_atomic,
                           float* grad_members, const int32_t* members, int n_members, int32_t* status, void* stream);
int ani_b200_dispersion_d3_cells(const ani_d3_params* params, const float* tables, const ani_grid* grid,
                                 const int32_t* bin_start, const float* spos, const int32_t* sorted_orig, int n, int lo,
                                 int hi, int n_conf, int n_per_conf, float skin, float* cn, float* dedcn, float* atomic,
                                 double* energies, float* grad_coords, double* virial, float* member_atomic,
                                 float* grad_members, const int32_t* members, int n_members, int32_t* status,
                                 const float* lattice, void* stream);
/*    The same term over a caller-supplied HALF pair list (conventions of ani_b200_pair_potential_pairs; cutoff_fn 2 =   */
/*    no envelope and no cutoff).  A pair that touches a ghost atom counts half in the energy and fully in the           */
/*    coordination numbers.  cn, dedcn: f32[n] scratch (zeroed here; dedcn may be NULL without grad_coords).  Three       */
/*    launches (two without grad_coords), float atomics; not the hot path.                                              */
int ani_b200_dispersion_d3_pairs(const ani_d3_params* params, const float* tables, const int32_t* species,
                                 const int64_t* idx0, const int64_t* idx1, const float* distances,
                                 const float* diff_vectors, const uint8_t* ghost_flags, int64_t num_pairs, int n_conf,
                                 int n_per_conf, float* cn, float* dedcn, float* atomic, double* energies,
                                 float* grad_coords, void* stream);

/* 4b. The same AEV kernels fed by an externally supplied HALF pair list (the reference's    */
/*    Neighbors tuple; AEVComputer.compute_from_neighbors, aev/_computer.py:251-272 ->          */
/*    cuaev::run_with_half_nbrlist, csrc/aev.cu:1128-1208,1779-1866).  ani_b200_pairs_to_rows     */
/*    expands the list into per-atom rows (both directions): row_start i32[n+1], row_j i32[2P],  */
/*    row_d f32[2P][4] = (r_j - r_i, R); scratch i32[2n].  diff_vectors follow the reference:     */
/*    x[idx0] - x[idx1] + shift.  The *_rows entry points then take any `grid` whose n_real == n  */
/*    and an `spos` that only needs the species in .w (atoms in input order, padding = -1).       */
/*    Gradients go to the coordinates only, as in csrc/cuaev.cpp:158-163.                          */
int ani_b200_pairs_to_rows(const int64_t* idx0, const int64_t* idx1, const float* diff_vectors,
                           int64_t num_pairs, int n, int nbr_cap, int32_t* row_start,
                           int32_t* row_j, float* row_d, int32_t* scratch_i32, int32_t* status,
                           void* stream);
/* 4c. FULL neighbour list with ghost atoms, as MD engines hand it over (LAMMPS pair style, pmemd): replaces   */
/*    cuaev::run_with_full_nbrlist (csrc/cuaev.cpp:225-246, csrc/aev.cu:1048-1126,1868-1956;                      */
/*    aev/_computer.py:409-438).  coords f32[n_all][3] hold local AND ghost atoms (ghosts at their image          */
/*    positions, no cell), ilist i32[n_i] the atoms whose AEV is wanted, numneigh i32[n_i] their neighbour         */
/*    counts, jlist i32[sum numneigh] the neighbours of ilist[0], ilist[1], ... one after the other (built with    */
/*    cutoff + skin: entries beyond `cutoff` are screened out here).  Output: the per-atom rows of 4b              */
/*    (row_start i32[n_all+1], row_j / row_d with capacity sum(numneigh)); atoms not in ilist get empty rows, i.e.  */
/*    all-zero AEVs, as in the reference.  scratch i32[n_all + n_i + 1].  Feed the result to                         */
/*    ani_b200_aev_forward_rows / _backward_rows (gradients reach local and ghost coordinates alike).                */
int ani_b200_full_nbrlist_to_rows(const float* coords, int n_all, const int32_t* ilist, const int32_t* numneigh,
                                  const int32_t* jlist, int n_i, float cutoff, int nbr_cap, int32_t* row_start,
                                  int32_t* row_j, float* row_d, int32_t* scratch_i32, int32_t* status, void* stream);
int ani_b200_aev_forward_rows(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                              const int32_t* row_start, const int32_t* row_j, const float* row_d,
                              int n, const int32_t* row_of, float* aev, int ldx, int layout,
                              int nbr_cap, int32_t* status, void* stream);
int ani_b200_aev_backward_rows(const ani_aev_params* params, const ani_grid* grid, const float* spos,
                               const int32_t* sorted_orig, const int32_t* row_start,
                               const int32_t* row_j, const float* row_d, int n, const int32_t* row_of,
                               const float* grad_aev, int ldx, int nbr_cap, float* grad_coords,
                               int32_t* status, void* stream);

/* 3c. Verlet-skin reuse of a bucket grid (neighbors.py:759-884, VerletCellList).  Build the grid  */
/*     with cutoff + skin (ani_b200_prepare_step / ani_b200_build_cells), then                      */
/*       mode 0  right after the build: remember the binned positions (ref_pos f32[n][4]) and the   */
/*               lattice vector that wrapped every atom into the cell (ref_shift f32[n][4]);        */
/*       mode 1  on later steps INSTEAD of a rebuild: spos = new coords + ref_shift in the same     */
/*               sorted order (every other output of the build stays valid), zero-fills             */
/*               zero_f32[0..count) like the fused preparation, and ORs into `moved` (i32[1],       */
/*               cleared by the caller) bit 0 if any atom is more than skin/2 from its binned        */
/*               position (the step is invalid), bit 1 if any is beyond 70 % of that (a hint to      */
/*               rebuild before the next step).                                                       */
/*     While bit 0 of `moved` stays 0 every pair within the true cutoff is still inside the 27 buckets around */
/*     an atom and the AEV kernels (which screen with the true cutoff and the current positions)    */
/*     give exactly the result of a rebuild; when it is raised the step must be redone after a      */
/*     rebuild.  aev_blocks (or NULL): the block list of the build, its "composition changed" flag  */
/*     is cleared in mode 1.                                                                          */
int ani_b200_verlet_positions(int mode, const float* coords, const ani_grid* grid,
                              const int32_t* sorted_orig, int n, float skin, float* spos, float* ref_pos,
                              float* ref_shift, int32_t* moved, float* zero_f32, int zero_f32_count,
                              int32_t* aev_blocks, int ldx, void* stream);

/* 3b. Fused per-step preparation: build_cells + species_layout + active_aev_blocks in ONE launch     */
/*     (a persistent grid with device-wide barriers between its five phases) instead of twelve       */
/*     (same outputs, same determinism; what the fused engine calls).                                 */
/*     Also zero-fills zero_f32[0..count) (the force accumulator) and zero_f64[0..count) (the      */
/*     conformer energies) so that no separate memset launches are needed.                          */
/*     bucket_species (or NULL): i32[max_bins][8], per bucket the offset of its first atom of species >= s */
/*     (buckets are species-sorted), consumed by ani_b200_aev_forward.  bucket_ranges and bucket_species  */
/*     are filled in grid modes 0 and 2 (ignored in mode 1).  Mode 2 runs the persistent-grid or the  */
/*     five-launch form (the thread-block-cluster form is mode 0 only); same outputs.               */
/*     scratch_i32: 3 n + max_bins + 4 + (max(1, ceil((hi-lo)/256)) + 2) * ANI_MAX_SPECIES + 32 ints (an empty     */
/*     slice still takes one layout chunk), ZERO at allocation (two of them are the state of the device-wide      */
/*     barrier of the single-launch preparation).                                                               */
int ani_b200_prepare_step(const float* coords, const int32_t* species, int n_conf, int n_per_conf,
                          const float* cell, int pbc, int mode, float cutoff, int max_bins, ani_grid* grid,
                          int32_t* bin_start, int32_t* sorted_orig, int32_t* orig_to_sorted, float* spos,
                          int32_t* sbin, float* bucket_ranges, int lo, int hi, int num_species, int rows_cap,
                          int32_t* row_of, int32_t* row_atom, int32_t* tile_species, int32_t* layout_info,
                          int n_shf_r, int angular_sub, int out_dim, int ldx, int ang_pad, int32_t* aev_blocks,
                          float* zero_f32, int zero_f32_count, double* zero_f64, int zero_f64_count,
                          int32_t* bucket_species, int32_t* scratch_i32, int32_t* status, void* stream);

/* 3e. The same preparation in grid mode 3: a periodic batch with ONE CELL PER CONFORMER (the frames of an NPT      */
/*     trajectory, a screened dataset).  Arguments of ani_b200_prepare_step with mode == 3 (else                     */
/*     ANI_ERR_UNSUPPORTED), pbc == 1, n_conf + 1 <= max_bins, and                                                   */
/*       cell     device f32[n_conf][9], rows of every 3x3 block are that conformer's lattice vectors              */
/*       lattice  device f32[n_conf][ANI_LATTICE_STRIDE] (out, not NULL): per conformer {cell[9], inverse[9]}, the    */
/*                inverse computed in double and rounded; read by ani_b200_aev_forward_cells / _backward_cells.    */
/*     Buckets are conformer-major as in mode 2 (bucket c * nb + local) with sub-grid dims common to all            */
/*     conformers: per axis the minimum over the conformers of floor(perpendicular width / (cutoff + 1e-5)),        */
/*     capped so that nb <= (max_bins - 1) / n_conf.  Every atom is wrapped, and every image shift of the range     */
/*     table is taken, in its own conformer's lattice.  A conformer whose cell is thinner than the cutoff raises    */
/*     ANI_STATUS_CELL_TOO_SMALL.  With C equal cells every output equals that of mode 2 on the shared cell.       */
/*     Runs the persistent-grid form or the five-launch form (+ one single-CTA setup launch); same outputs.        */
int ani_b200_prepare_step_cells(const float* coords, const int32_t* species, int n_conf, int n_per_conf,
                                const float* cell, int pbc, int mode, float cutoff, int max_bins, ani_grid* grid,
                                int32_t* bin_start, int32_t* sorted_orig, int32_t* orig_to_sorted, float* spos,
                                int32_t* sbin, float* bucket_ranges, int lo, int hi, int num_species, int rows_cap,
                                int32_t* row_of, int32_t* row_atom, int32_t* tile_species, int32_t* layout_info,
                                int n_shf_r, int angular_sub, int out_dim, int ldx, int ang_pad, int32_t* aev_blocks,
                                float* zero_f32, int zero_f32_count, double* zero_f64, int zero_f64_count,
                                int32_t* bucket_species, int32_t* scratch_i32, int32_t* status, float* lattice,
                                void* stream);

/* Timing experiments only: the first 4 CTAs of the next `launches` tensor-core GEMM launches    */
/* write clock64 stamps [launch][cta 4][tile 8][role 3: producer, MMA, epilogue][4] into buf       */
/* (device memory, launches*384 int64).  NULL switches it off.  No reference counterpart.           */
int ani_b200_debug_gemm_trace(long long* buf, int launches);

/* Timing experiments only: the CTA-staged AEV forward kernel writes per-phase clock64 cycles and    */
/* %globaltimer / clock64 stamps, 16 int64 per record, into buf (device memory): one record per atom */
/* (index - lo).  NULL switches it off.                                                              */
/* ANI_ERR_UNSUPPORTED unless the library was built with -DANI_AEV_FWD_TRACE=1 (build variant      */
/* "aevtrace").  No reference counterpart.                                                            */
int ani_b200_debug_aev_trace(long long* buf);

/* 5. Reference-format half neighbour list (neighbors.py:13-18) from the bucket grid.       */
/*    Two calls: count (fills pair_start i32[n+1], exclusive scan, total in pair_start[n]),  */
/*    then fill with capacity `cap` pairs.  indices are flat INPUT indices, idx0 < idx1       */
/*    except for self-image pairs; diff = x[idx0] - x[idx1] + shift (neighbors.py:107-111).   */
int ani_b200_half_neighbor_count(const ani_grid* grid, const int32_t* bin_start, const float* spos,
                                 const int32_t* sbin, const int32_t* sorted_orig, int n,
                                 float cutoff, int32_t* pair_start, void* stream);
int ani_b200_half_neighbor_fill(const ani_grid* grid, const int32_t* bin_start, const float* spos,
                                const int32_t* sbin, const int32_t* sorted_orig, int n, float cutoff,
                                const int32_t* pair_start, int64_t cap, int64_t* idx0, int64_t* idx1,
                                float* distances, float* diff_vectors, int32_t* status, void* stream);

/* 6. Ensemble MLP forward + backward-to-input on the species-grouped AEV matrix.           */
/*    Layer widths: in -> h1 -> h2 -> h3 -> 1, the activation after the three hidden layers: */
/*    ani_mlp_model::activation = ANI_ACT_CELU: CELU(celu_alpha), every layer with biases;    */
/*                                ANI_ACT_GELU: GELU (exact erf form), no biases (the packer  */
/*                                passes zeros in b1..b4, which the GELU kernels never read). */
/*    Any other value: ANI_ERR_BAD_ARG from every entry point of this section.                */
/*    "Tiled operand" layout (both GEMM operands; fp32 accuracy on the tensor cores from 16-bit    */
/*    pieces, see ani_b200_operand_format): every value x of an operand with power-of-two scale s   */
/*    is stored as P pieces with s*x = p1 + ... + pP, each rounded to nearest:                       */
/*      P = 2 IEEE half pieces (default build; 4 B/element; s = 64 for AEVs/activations, 4096 for    */
/*            gradients, ani_mlp_species::w_scale for weights; |s*x| must stay below 65504, else     */
/*            ANI_STATUS_OPERAND_RANGE is raised and the results are inf/NaN),                       */
/*      P = 3 bfloat16 pieces (-DANI_OPND_FP16X2=0; 6 B/element; s = 1).                             */
/*    * A operand / activation matrix [rows][cols] (rows % 128 == 0, cols % 32 == 0):                */
/*        [row tile of 128][32-column block][p1: 128 rows x 64 B | p2 (| p3)]    (16 / 24 KB blocks) */
/*    * B operand of a layer GEMM  C[rows, N] = A[rows, K] x W  (W given as B[N][K], N % 32 == 0,  */
/*      K padded to a multiple of 32 with zeros):                                                  */
/*        [member][n tile (256 rows, the last one shorter)][32-column block][p1 bn x 64 B | p2 (| p3)] */
/*    In both, every 8-row x 64-byte group is in the wgmma SWIZZLE_64B order (16-byte chunk c      */
/*    of row r sits at chunk position c ^ ((r >> 1) & 3)), i.e. exactly the shared-memory image    */
/*    a K-major UMMA descriptor expects: one K-block of one tile is a contiguous byte range        */
/*    that a single cp.async.bulk (TMA) moves into shared memory.  Hidden widths that are not       */
/*    multiples of 32 are zero-padded by the packer (zero weights and biases: CELU(0) = GELU(0) = 0; */
/*    GELU'(0) = 1/2 in the padded columns meets the zero rows of the transposed weights).         */
#define ANI_ACT_CELU 0
#define ANI_ACT_GELU 1
typedef struct ani_mlp_species {
  int32_t h1, h2, h3, pad_;
  float w_scale[4];  /* [0..2]: power-of-two scale the packer multiplied W1, W2, W3 by (fp16 pieces) */
  const float* b1;   /* [M*h1]                                                                  */
  const float* b2;   /* [M*h2]                                                                  */
  const float* b3;   /* [M*h3]                                                                  */
  const float* w4;   /* [M][h3]                                                                 */
  const float* b4;   /* [M]                                                                     */
  const void* t_f1;  /* forward  layer 1: per member B = W1_m [h1][in_dim -> ldx]               */
  const void* t_f2;  /* forward  layer 2: per member B = W2_m [h2][h1]                          */
  const void* t_f3;  /* forward  layer 3: per member B = W3_m [h3][h2]                          */
  const void* t_b3;  /* backward layer 3: per member B = W3_m^T [h2][h3]                        */
  const void* t_b2;  /* backward layer 2: per member B = W2_m^T [h1][h2]                        */
  const void* t_b1;  /* backward layer 1: B = W1^T [ldx][M*h1]                                  */
} ani_mlp_species;

typedef struct ani_mlp_model {
  int32_t num_species, num_members, in_dim, ldx;
  int32_t h1_max, h2_max, h3_max;
  int32_t activation;                  /* ANI_ACT_CELU or ANI_ACT_GELU                          */
  float celu_alpha;                    /* ANI_ACT_CELU only                                     */
  float member_scale[ANI_MAX_MEMBERS]; /* d(output)/d(member energy): 1/M_active or 0       */
  ani_mlp_species sp[ANI_MAX_SPECIES];
  /* optional device scratch, sum over the species of ldx * (M * h1 / 32) * 2 * P * 32 bytes (the size of the t_b1   */
  /* operands together), or NULL: every step gathers the LIVE column blocks of the layer-1 backward operands into   */
  /* it (ani_b200_zero_live_blocks / ani_b200_mlp_step / ani_b200_mlp_backward), so that the GEMM moves one         */
  /* K-block of them with one bulk copy.  No state is carried between steps; one step at a time per model.          */
  void* b1_compact;
} ani_mlp_model;

/* 6a. Model-pack time: plain fp32 weights -> the tiled B operand above (one launch per operand; `batch`   */
/*     operands of the same shape, e.g. the members of an ensemble, src/dst `*_batch_stride` elements/bytes     */
/*     apart).  src is [n][ld_src] (B[n][k] = src[n][k]) or, with transpose != 0, [k][ld_src] (B[n][k] =       */
/*     src[k][n]: the backward operands are the transposed weights); n % 32 == 0; K is zero-padded to a        */
/*     multiple of 32; every value is multiplied by the power-of-two `scale` first.                             */
/*     dst: batch * n * ceil32(k) * 2 * P bytes.  Replaces BmmLinear.__init__ (nn/_infer.py:171-203), the       */
/*     reference's own inference-time re-layout of the weights.                                                 */
int ani_b200_pack_b_operand(const float* src, int n, int k, int ld_src, int transpose, float scale, int batch,
                            long long src_batch_stride, void* dst, long long dst_batch_stride, void* stream);

/*    x            tiled operand, in: AEVs (ani_b200_aev_forward layout 1), 2*P*rows_cap*ldx bytes */
/*    dx           f32[rows_cap][ldx] plain rows, out: dE/dAEV (may be NULL if !want_backward)  */
/*    row_atom / layout_info: outputs of ani_b200_species_layout                                */
/*    aev_blocks   output of ani_b200_active_aev_blocks or NULL (= every column is live).       */
/*                 With a block list, layer 1 skips the dead K-blocks and dE/dAEV is written     */
/*                 only for the live column blocks (the others keep their previous content).     */
/*    act1/2/3     tiled operands, 2*P*rows_cap*M*h{1,2,3}_max bytes (activations, then gradients) */
/*                 GELU model: act1 / act2 are twice that size.  The first half is the activation   */
/*                 operand as above; the second, the derivative operand of the same shape directly  */
/*                 behind it, receives GELU'(z) of every element from the forward (want_backward    */
/*                 != 0 only; at the value scale), which the backward multiplies by: GELU cannot be */
/*                 recovered from its output as CELU' is.                                           */
/*    e_member     f32[M][rows_cap]     per-member atomic energies                               */
/*    status       i32[1] device word, ANI_STATUS_OPERAND_RANGE is OR-ed in (may be NULL)        */
int ani_b200_mlp_forward_backward(const ani_mlp_model* model, const void* x, float* dx, int rows_cap,
                                  const int32_t* row_atom, const int32_t* layout_info,
                                  const int32_t* aev_blocks, void* act1, void* act2, void* act3,
                                  float* e_member, int want_backward, int32_t* status, void* stream);

/*    The same work as two calls, so that a caller can run independent work beside the backward      */
/*    GEMMs (engine.py: ani_b200_reduce_energies only needs e_member, i.e. the forward half) and      */
/*    zero dE/dAEV ahead of time on another stream:                                                    */
/*      ani_b200_mlp_forward       layers 1-3 + final layer + gradient seed (act3)                    */
/*      ani_b200_zero_live_blocks  dx[rows][live column blocks] = 0 (the layer-1 backward accumulates  */
/*                                 the members into dx; only needed when num_members > 1)              */
/*      ani_b200_mlp_backward      the three backward-to-input GEMMs; dx_zeroed != 0: the caller has   */
/*                                 already run ani_b200_zero_live_blocks for this step                 */
int ani_b200_mlp_forward(const ani_mlp_model* model, const void* x, int rows_cap, const int32_t* row_atom,
                         const int32_t* layout_info, const int32_t* aev_blocks, void* act1, void* act2,
                         void* act3, float* e_member, int want_backward, int32_t* status, void* stream);
int ani_b200_zero_live_blocks(const ani_mlp_model* model, float* dx, const int32_t* layout_info,
                              const int32_t* aev_blocks, void* stream);
int ani_b200_mlp_backward(const ani_mlp_model* model, float* dx, int rows_cap, const int32_t* row_atom,
                          const int32_t* layout_info, const int32_t* aev_blocks, void* act1, void* act2,
                          void* act3, int dx_zeroed, int32_t* status, void* stream);

/*    The same six GEMMs as ONE persistent launch (csrc/gemm_tc.cuh): the (layer, row tile, member, column        */
/*    tile) units form one list and the launch boundaries are replaced by data-flow waits on per-(layer, row tile,   */
/*    member) completion counters -- no ramp / tail per layer, one tile-count quantisation for the whole step, and   */
/*    at small row counts (multi-GPU shards) no per-launch floor.  sync_i32: 6 * (rows_cap / 128) * ANI_MAX_MEMBERS  */
/*    ints of scratch (zeroed by the call).  Same arguments and results as ani_b200_mlp_forward_backward otherwise.  want_backward == 2:          */
/*    PER-MEMBER gradients (arch.py:403-436, members_forces): dx is f32[M][rows_cap][ldx] and member m's slab receives   */
/*    d(member_scale[m] * e_m)/dAEV by plain stores (no sum over the members, no zero-fill needed).                      */
/*    ani_b200_mlp_step runs a step as ani_b200_mlp_step_windows(model, rows_cap) launches of the data-flow kernel, */
/*    one per window of the row tiles (all six phases of a window, then the next), sized so that a window's         */
/*    activations stay in the L2 between the phase that writes them and the phases that read them.                  */
int ani_b200_mlp_step_windows(const ani_mlp_model* model, int rows_cap);
int ani_b200_mlp_step(const ani_mlp_model* model, const void* x, float* dx, int rows_cap, const int32_t* row_atom,
                      const int32_t* layout_info, const int32_t* aev_blocks, void* act1, void* act2, void* act3,
                      float* e_member, int want_backward, int32_t* sync_i32, int32_t* status, void* stream);

/*    The same step with gradients (want_backward == 1) as one launch that keeps every intermediate of a      */
/*    (row tile, member) chain in shared memory (csrc/mlp_resident.cuh): act1 / act2 receive the activations   */
/*    a1 / a2 (tiled, scaled like the forward's), e_member and dx as above; no act3, no gradient pieces in     */
/*    global memory, no counters.  GELU model: act1 / act2 receive d1 = GELU'(z1) / d2 = GELU'(z2) instead of   */
/*    a1 / a2 (same tiled layout and scale, same size as for CELU: no derivative operand behind them).         */
/*    ANI_ERR_UNSUPPORTED in the 3 x bf16 build and for models with a hidden width above 256.                  */
int ani_b200_mlp_step_resident(const ani_mlp_model* model, const void* x, float* dx, int rows_cap,
                               const int32_t* row_atom, const int32_t* layout_info, const int32_t* aev_blocks,
                               void* act1, void* act2, float* e_member, int32_t* status, void* stream);

/*    The same launch with one dE/dAEV slab per member (the query-by-committee step, ani_b200_aev_backward_members):   */
/*    the arguments of ani_b200_mlp_step_resident plus slab_stride (floats, >= rows_cap * ldx).  Only the chains of    */
/*    the ACTIVE members (member_scale[m] != 0) run.  Active member m's slab, dx + m * slab_stride, f32[rows_cap][ldx], */
/*    receives d(member_scale[m] * e_m)/dAEV by plain stores in the rows of the row tiles of the layout (padding rows  */
/*    get zeros) and the live column blocks of aev_blocks (every column without a block list); no other column or row, */
/*    and no slab of an inactive member, is written.  No zero-fill is needed: ani_b200_aev_backward_members reads     */
/*    only the live blocks of active members' real rows.  e_member rows of inactive members are set to 0.  Same limits  */
/*    as ani_b200_mlp_step_resident (ANI_ERR_UNSUPPORTED in the 3 x bf16 build and above hidden width 256; there,     */
/*    ani_b200_mlp_step(..., want_backward = 2) provides the slabs); ANI_ERR_BAD_ARG without an active member.       */
int ani_b200_mlp_step_resident_members(const ani_mlp_model* model, const void* x, float* dx, long long slab_stride,
                                       int rows_cap, const int32_t* row_atom, const int32_t* layout_info,
                                       const int32_t* aev_blocks, void* act1, void* act2, float* e_member,
                                       int32_t* status, void* stream);

/* 7. Scatter per-member atomic energies back to input order and reduce per conformer.      */
/*      atomic_out f32[n] (mean over active members, 0 for padding; flat input order)         */
/*      member_atomic_out f32[M][n] or NULL                                                    */
/*      energies_out f64[n_conf]  NN energy + self energies (sae f64[num_species] or NULL)     */
/*    Only atoms whose sorted position is in lo..hi-1 contribute (others give 0), so the     */
/*    per-rank results of a sharded run add up to the full answer.                            */
int ani_b200_reduce_energies(const ani_mlp_model* model, const float* e_member, int rows_cap,
                             const int32_t* row_of, const int32_t* orig_to_sorted,
                             const int32_t* species, int n, int lo, int hi, int n_conf,
                             int n_per_conf, const double* sae, float* atomic_out,
                             float* member_atomic_out, double* energies_out, void* stream);

/* 7b. Atomic charges and dipoles of a charge model (ANIq / ANImbis), one launch, one CTA per conformer.              */
/*    q_raw        raw charges: with row_of / orig_to_sorted (outputs of the step preparation) the e_member row 0    */
/*                 f32[rows_cap] of a one-member charge network pass, read at row_of[orig_to_sorted[a]]; with both   */
/*                 NULL, f32[n] in flat input order                                                                 */
/*    species      i32[n] element indices, -1 = padding;  coords f32[n][3] in flat INPUT order (not wrapped)         */
/*    weights      HOST f32[num_species] normaliser weights (may be NULL if !normalize); scale_by_q2: w_i = W[e_i]   */
/*                 * q_raw_i^2 (ChargeNormalizer's scale_weights_by_charges_squared); normalize == 0: q = q_raw      */
/*                 (BaseChargeNormalizer)                                                                           */
/*    total_charge Q: normalised charges are q_i = q_raw_i + (Q - sum q_raw) w_i / sum w                          */
/*    masses       HOST f32[num_species], needed only for frame 0                                                    */
/*    frame        dipole reference point: 0 centre of mass, 1 centre of geometry (real atoms), 2 origin           */
/*    charges_out  f32[n], input order, 0 for padding                                                                */
/*    dipoles_out  f64[n_conf][3] = sum_i q_i (r_i - r_ref) over the real atoms, in e * Angstrom, or NULL            */
/*    Float64 sums in a fixed order (no atomics): repeated runs give identical bits.                                */
int ani_b200_charges(const float* q_raw, const int32_t* row_of, const int32_t* orig_to_sorted, const int32_t* species,
                     const float* coords, int n_conf, int n_per_conf, const float* weights, int num_species,
                     int scale_by_q2, int normalize, double total_charge, const float* masses, int frame,
                     float* charges_out, double* dipoles_out, void* stream);

/* 8. Multi-GPU: one-shot all-reduce of the per-rank partial forces / energies over NVLink peer memory.   */
/*    The path shards by central atom (one process per GPU); every rank accumulates dE_owned/dx_j into a      */
/*    full-length f32[n_f32] buffer and its share of the conformer energies into f64[n_f64].  Those partial     */
/*    buffers live in CUDA-IPC memory owned by the communicator (the ONE place where this library allocates:    */
/*    IPC-exportable memory must come from cudaMalloc) and are mapped by every peer; ani_b200_comm_allreduce     */
/*    launches ONE kernel: flag barrier in peer memory, every rank sums the W partials in rank order (bitwise      */
/*    identical totals everywhere) into its own out buffers, flag barrier.  Graph-capturable; epochs advance on     */
/*    the device.  The reference has no collective (SURVEY.md 2.1) -- this replaces the NCCL all-reduce of         */
/*    round 1 (parallel.py).  Set-up: create on every rank, exchange the 64-byte handles by any host channel        */
/*    (torch.distributed all_gather here), connect with the W handles in rank order.  world <= 8, one node.          */
/*    error_word (device i32): raised by the kernel if a peer does not arrive within ~10 s (no hang).               */
int ani_b200_comm_create(int rank, int world, long long n_f32, long long n_f64, void** comm_out);
int ani_b200_comm_handle(void* comm, void* handle64);
int ani_b200_comm_connect(void* comm, const void* handles);
int ani_b200_comm_buffers(void* comm, float** partial_f32, double** partial_f64, int32_t** error_word);
int ani_b200_comm_allreduce(void* comm, float* out_f32, double* out_f64, void* stream);
int ani_b200_comm_destroy(void* comm);

/* 9. Analytic Hessians of open systems (csrc/hessian.cu), after a step with gradients (grid mode 0 or 1, one rank):  */
/*    they read what it left behind -- sorted positions, nbr_cnt / nbr_list, row_of, sorted_orig, the tiled AEVs x and */
/*    the member-weighted dE/dAEV rows dx -- and change none of it.  Per central atom i with n_i = min(nbr_cnt, cap)   */
/*    neighbour words, one block B_i (f32, 3 n_i x 3 n_i, row / column 3 n + c = component c of r_n - r_i of          */
/*    neighbour n) collects the second derivatives of i's energy terms with respect to those relative vectors:        */
/*      ani_b200_hessian_jacobian   the AEV Jacobian rows J_i (row 3 n + c = dA_i / d(r_n - r_i)_c, f32[ldx] in the     */
/*                                  internal column order of x / dx; the chunk's rows are zeroed first)              */
/*      ani_b200_hessian_network    B_i += J_i^T K_i J_i, K_i = sum over the members with member_scale[m] != 0 of      */
/*                                  member_scale[m] times the network Hessian at A_i: one fp32 primal pass per         */
/*                                  (atom, member), five tangent GEMMs over the rows and Zdot1 Deltadot1^T per atom.  */
/*                                  scratch: 4 rows hmax + n_slots 5 hmax floats, hmax = ani_b200_hessian_hidden_max  */
/*      ani_b200_hessian_geometric  with dx (pair_dev NULL): the Hessian of dx_i . A_i with dx_i held fixed; with a     */
/*                                  DEVICE copy of one ani_pair_params of kind 0 or 1 (dx NULL): the Hessian of its    */
/*                                  1/2 E(R) fc(R) per neighbour word within its cutoff                              */
/*      ani_b200_hessian_assemble   hess[conf][3 A][3 A] (f64, input atom order, accumulated; the caller zeroes it)    */
/*                                  += B_i mapped onto atoms {i} u nbrs(i): (j, k) += B, (i, k) and (j, i) -= the     */
/*                                  sums over j / k, (i, i) += the sum of B                                          */
/*    A chunk is a set of central atoms ("slots") processed together (device arrays):                                 */
/*      atom[n_slots]        sorted index of each slot's atom                                                         */
/*      row_off[n_slots]     first Jacobian row of the slot (3 n_i rows); slots of one species are contiguous and     */
/*                           every species segment starts at a multiple of ANI_HESSIAN_ROW_ALIGN                     */
/*      block_off[n_slots]   first float of B_i in `blocks`                                                          */
/*      row_slot[rows]       slot of each row, -1 for the rows between the segments                                   */
/*      tile_species[rows / ANI_HESSIAN_ROW_ALIGN]  species of each row tile                                           */
/*      rows                 multiple of ANI_HESSIAN_ROW_ALIGN;  max_count: largest n_i of the chunk                    */
/*    `blocks` must be zeroed before the network and geometric calls of a chunk, which add into it.                   */
#define ANI_HESSIAN_ROW_ALIGN 64
typedef struct ani_hessian_chunk {
  const int32_t* atom;
  const int32_t* row_off;
  const long long* block_off;
  const int32_t* row_slot;
  const int32_t* tile_species;
  int32_t n_slots, rows, max_count, pad_;
} ani_hessian_chunk;
/*    Plain fp32 weights of every member, per species, in the padded widths of ani_mlp_species (h1, h2, h3):        */
/*      w1 [M][h1][ldx] (internal column order), w2 [M][h2][h1], w3 [M][h3][h2]; biases and w4 from ani_mlp_species.  */
typedef struct ani_hessian_weights {
  const float* w1[ANI_MAX_SPECIES];
  const float* w2[ANI_MAX_SPECIES];
  const float* w3[ANI_MAX_SPECIES];
} ani_hessian_weights;
int ani_b200_hessian_hidden_max(const ani_mlp_model* model);
int ani_b200_hessian_jacobian(const ani_aev_params* params, const float* spos, const int32_t* nbr_cnt,
                              const int32_t* nbr_list, int cap, const ani_hessian_chunk* chunk, float* jac, int ldx,
                              void* stream);
int ani_b200_hessian_network(const ani_mlp_model* model, const ani_hessian_weights* weights, const void* x,
                             const int32_t* row_of, const float* spos, const int32_t* nbr_cnt, int cap,
                             const ani_hessian_chunk* chunk, const float* jac, float* scratch, float* blocks,
                             void* stream);
int ani_b200_hessian_geometric(const ani_aev_params* params, const float* spos, const int32_t* nbr_cnt,
                               const int32_t* nbr_list, int cap, const int32_t* row_of, const float* dx, int ldx,
                               const ani_pair_params* pair_dev, const ani_hessian_chunk* chunk, float* blocks,
                               void* stream);
int ani_b200_hessian_assemble(const int32_t* nbr_cnt, const int32_t* nbr_list, int cap, const int32_t* sorted_orig,
                              const ani_hessian_chunk* chunk, const float* blocks, int n_per_conf, double* hess,
                              void* stream);

/* 10. Molecular dynamics on the device (csrc/md.cu): velocity Verlet (NVE), BAOAB Langevin (NVT) and Langevin with   */
/*    stochastic cell rescaling (NPT) integrators whose state stays in device memory, so that K whole MD steps          */
/*    (integrator + force step) capture into one CUDA graph.                                                          */
/*    Units: A, fs, amu, Hartree, K.  The caller owns every buffer (ani_md_state, device pointers unless noted):       */
/*      x, v        f64[n][3] master positions (unwrapped, input order) and velocities (A / fs)                         */
/*      inv_mass    f64[n] 1 / mass (1 / amu); 0 for padding atoms, which never move                                  */
/*      params      f64[n_conf][ANI_MD_PARAMS] per conformer: dt (fs), temperature (K), friction (1 / fs), the energy  */
/*                  QBC and the force relative-stdev stop thresholds (+inf: never), 3 N_real, two unused               */
/*      counter     i64[2] step counter t (counter[0]; counter[1] is the launches' own copy)                           */
/*      stop_step   i64[n_conf] -1 while running, else the step at which the conformer stopped                         */
/*      trigger     f64[2][n][3] x, v of a conformer at its stop step (written then only), or NULL                     */
/*      thermo      f64[thermo_rows][n_conf][ANI_MD_THERMO]: step t's record {t, E_pot, E_kin (Hartree), T (K)} goes    */
/*                  to row t % thermo_rows; T = 2 E_kin / (3 N_real k_B)                                                */
/*      frames      f64[frame_slots][1 + frame_velocities][n][3]: x (and v) of step t, where t % record_every == 0, in  */
/*                  slot (t / record_every) % frame_slots; unused with record_every == 0                              */
/*      partials    f64[n_conf][ceil(n_per_conf / ANI_MD_BLOCK)][2] scratch of ani_b200_md_step                        */
/*      seed        key of the Langevin noise;  accel = Hartree / (amu A^2) in fs^-2;  kb = k_B in Hartree / K         */
/*  ani_b200_md_init   per conformer, with zero_momentum: v -= total momentum / total mass (real atoms); then the      */
/*                     f32 coords (flat input order) of x, wrapped into the cell: cell_mode 0 open, 1 one cell f32[9]   */
/*                     (rows are lattice vectors), 2 one cell per conformer f32[n_conf][9].  One launch.               */
/*  ani_b200_md_step   after the force step at x(t) (grad f32[n][3] dE/dx, energies f64[n_conf]), two launches: the   */
/*                     final half kick B(dt/2) giving v(t) (none at t = 0: v(0) is the initial velocity), the thermo    */
/*                     record and frame of step t, the stop check, then B(dt/2) A(dt) (ANI_MD_VERLET) or              */
/*                     B(dt/2) A(dt/2) O(dt) A(dt/2) (ANI_MD_LANGEVIN, O: v = c v + sqrt((1 - c^2) k_B T / m) xi,      */
/*                     c = exp(-friction dt), xi = ani_b200_md_noise(seed, t)) to x(t+1), the f32 coords of x(t+1)      */
/*                     (wrapped into `cell` f32[9] when not NULL), and t += 1.  Stop check (qbc f64[n_conf] and          */
/*                     force_stdev f32[n], the query-by-committee step's energy QBC and force_relative_stdev, both or  */
/*                     neither): a running conformer whose qbc or largest force_stdev exceeds its threshold stops at     */
/*                     t: stop_step = t, trigger = x(t), v(t); its x and v never change again.  Sums are float64 in a   */
/*                     fixed order: the same state and forces give the same bits.  n_conf > 65535 or n_conf n_per_conf  */
/*                     > INT_MAX: ANI_ERR_UNSUPPORTED (before any CUDA call).                                          */
/*  ani_b200_md_step_cells  the same with one cell per conformer: the lattice table of grid mode 3                     */
/*                     (f32[n_conf][ANI_LATTICE_STRIDE], written by ani_b200_prepare_step_cells) in place of `cell`.    */
/*  ani_b200_md_noise  out f64[n][3]: the standard normals the O step of step `step` draws for atoms 0..n-1 (flat index */
/*                     over the conformers): Philox4x32-10 keyed on the seed, counter (step, atom, component), Box-Muller. */
/*  ani_b200_md_step_npt  ani_b200_md_step (ANI_MD_LANGEVIN only, no stop check) with isotropic stochastic cell        */
/*                     rescaling (Bernetti & Bussi, J. Chem. Phys. 153, 114107 (2020)), every conformer fully periodic.  */
/*                     With h(t) the master cell, V = |det h|, K = E_kin(t), W = the virial of the force step at x(t)    */
/*                     (its slots summed in a fixed order), T, dt from params and P0, tau_p, beta_T from baro->params:    */
/*                       P_int = (2 K - tr W) / (3 V)                                                                 */
/*                       de = -(beta_T / tau_p) (P0 - P_int) dt + sqrt(2 k_B T beta_T dt / (V tau_p)) xi  (de = d ln V)  */
/*                       mu = exp(de / 3);  after B A O A:  x(t+1) = mu x',  v <- v / mu,  h(t+1) = mu h(t)           */
/*                     xi = ani_b200_md_cell_noise(seed, t)[c].  The f32 coords of x(t+1) are wrapped into the           */
/*                     float32-rounded h(t+1), which is written to cell_out for the next force step (never read by this   */
/*                     launch).  ani_md_barostat (device pointers; units A, fs, Hartree):                                 */
/*                       master       f64[2][n_conf][9] master cell rows by step parity: step t reads slot t % 2 and      */
/*                                    writes slot (t + 1) % 2                                                          */
/*                       params       f64[n_conf][ANI_MD_BARO_PARAMS]: P0 (Hartree / A^3), tau_p (fs), beta_T (A^3 / Hartree) */
/*                       cell_out     f32 cell rows of conformer c at cell_out + c * cell_stride (>= 9): the cell the      */
/*                                    next preparation reads (the workspace's cell, or its cells of grid mode 3)          */
/*                       virial       f64[n_conf][virial_slots][9] the force step's virial slots (its W_ab partial sums)   */
/*                       record       f64[thermo_rows][n_conf][ANI_MD_BARO]: {V (A^3), P_int (Hartree / A^3)} of step t,   */
/*                                    in row t % thermo_rows, beside the thermo record                                 */
/*                       frame_cells  f64[frame_slots][n_conf][9] h(t) of each frame (not NULL with record_every > 0)      */
/*  ani_b200_md_cell_noise  out f64[n_conf]: the standard normals xi of the cell rescaling of step `step`: Philox      */
/*                     counter (step, conformer, component 3), a counter no atom draws.                                  */
#define ANI_MD_BLOCK 256
#define ANI_MD_PARAMS 8
#define ANI_MD_THERMO 4
#define ANI_MD_BARO_PARAMS 3
#define ANI_MD_BARO 2
#define ANI_MD_VERLET 0
#define ANI_MD_LANGEVIN 1
typedef struct ani_md_state {
  double* x;
  double* v;
  const double* inv_mass;
  const double* params;
  long long* counter;
  long long* stop_step;
  double* trigger;
  double* thermo;
  double* frames;
  double* partials;
  unsigned long long seed;
  double accel, kb;
  int32_t n_conf, n_per_conf, integrator, thermo_rows, record_every, frame_slots, frame_velocities, pad_;
} ani_md_state;
int ani_b200_md_init(const ani_md_state* state, const float* cells, int cell_mode, int zero_momentum, float* coords,
                     void* stream);
int ani_b200_md_step(const ani_md_state* state, const float* grad, const double* energies, const double* qbc,
                     const float* force_stdev, const float* cell, float* coords, void* stream);
int ani_b200_md_step_cells(const ani_md_state* state, const float* grad, const double* energies, const double* qbc,
                           const float* force_stdev, const float* lattice, float* coords, void* stream);
int ani_b200_md_noise(unsigned long long seed, long long step, int n, double* out, void* stream);
typedef struct ani_md_barostat {
  double* master;
  const double* params;
  float* cell_out;
  const double* virial;
  double* record;
  double* frame_cells;
  int32_t cell_stride, virial_slots;
} ani_md_barostat;
int ani_b200_md_step_npt(const ani_md_state* state, const ani_md_barostat* baro, const float* grad,
                         const double* energies, float* coords, void* stream);
int ani_b200_md_cell_noise(unsigned long long seed, long long step, int n_conf, double* out, void* stream);

/* 11. Geometry optimisation on the device (csrc/opt.cu): FIRE (Bitzek et al., PRL 97, 170201 (2006)) as ASE's        */
/*    ase.optimize.FIRE defines it, without its downhill check, one independent optimisation per conformer.  The state */
/*    stays in device memory, so that K whole steps (FIRE + force step) capture into one CUDA graph, as in section 10.  */
/*    Units: A, eV, Hartree.  The caller owns every buffer (ani_opt_state, device pointers):                            */
/*      x, v        f64[n][3] master positions (unwrapped, input order) and FIRE velocities (eV / A x the time unit)     */
/*      force_scale f64[n] f = -dE/dx * force_scale: HARTREE_TO_EV for movable real atoms, 0 for fixed or padding atoms  */
/*      params      f64[n_conf][ANI_OPT_PARAMS] per conformer: dt0, maxstep (A), dtmax, Nmin, finc, fdec, astart, fa,  */
/*                  the fmax threshold (eV / A).  Not read by the validation of the entry points (device memory): the     */
/*                  caller keeps 0 < fdec < 1 <= finc, 0 < fa <= 1, dt0, maxstep, dtmax > 0 and fmax >= 0               */
/*      scalars     f64[2][n_conf][ANI_OPT_SCALARS] {dt, a, n} by step parity: step t reads slot t % 2 and writes slot    */
/*                  (t + 1) % 2                                                                                     */
/*      counter     i64[2] step counter t (counter[0]; counter[1] is the launches' own copy)                           */
/*      conv_step   i64[n_conf] -1 while the conformer runs, else the step at which it converged                        */
/*      record      f64[record_rows][n_conf][ANI_OPT_RECORD]: step t's record {t, E (Hartree), fmax (eV / A)} goes to    */
/*                  row t % record_rows                                                                              */
/*      partials    f64[n_conf][ceil(n_per_conf / ANI_MD_BLOCK)][4] scratch of ani_b200_opt_step                       */
/*  ani_b200_opt_init  with reset: v = 0 and the scalars of slot counter[0] % 2 = {dt0, astart, 0}; then the f32       */
/*                     coords of x, wrapped into the cell: cell_mode 0 open, 1 one cell f32[9], 2 one cell per          */
/*                     conformer f32[n_conf][9].  One launch.                                                         */
/*  ani_b200_opt_step  after the force step at x(t) (grad f32[n][3] dE/dx, energies f64[n_conf]), two launches, per    */
/*                     conformer with fmax(t) = max_i |f_i|:                                                           */
/*                       record {t, E, fmax(t)};  fmax(t) < threshold (and running): conv_step = t, and from then on    */
/*                       x, v, dt, a, n never change;  else P = f.v, F2 = f.f, V2 = v.v and                            */
/*                       t > 0, P > 0:  c1 = 1 - a, c2 = a sqrt(V2 / F2);  n > Nmin: dt = min(dt finc, dtmax), a *= fa; */
/*                                      n += 1                                                                       */
/*                       t > 0, P <= 0: c1 = c2 = 0, a = astart, dt *= fdec, n = 0                                   */
/*                       t = 0:         c1 = 1, c2 = 0                                                               */
/*                       v' = c1 v + (c2 + dt) f,  |dr| = dt sqrt(c1^2 V2 + 2 c1 (c2 + dt) P + (c2 + dt)^2 F2),        */
/*                       x(t+1) = x(t) + dt v' min(1, maxstep / |dr|)                                                   */
/*                     then the f32 coords of x(t+1) (wrapped into `cell` f32[9] when not NULL), and t += 1.  Sums are   */
/*                     float64 in a fixed order: the same state and forces give the same bits.                         */
/*  ani_b200_opt_step_cells  the same with one cell per conformer: the lattice table of grid mode 3                    */
/*                     (f32[n_conf][ANI_LATTICE_STRIDE], written by ani_b200_prepare_step_cells) in place of `cell`.    */
#define ANI_OPT_PARAMS 9
#define ANI_OPT_SCALARS 3
#define ANI_OPT_RECORD 3
typedef struct ani_opt_state {
  double* x;
  double* v;
  const double* force_scale;
  const double* params;
  double* scalars;
  long long* counter;
  long long* conv_step;
  double* record;
  double* partials;
  int32_t n_conf, n_per_conf, record_rows, pad_;
} ani_opt_state;
int ani_b200_opt_init(const ani_opt_state* state, const float* cells, int cell_mode, int reset, float* coords,
                      void* stream);
int ani_b200_opt_step(const ani_opt_state* state, const float* grad, const double* energies, const float* cell,
                      float* coords, void* stream);
int ani_b200_opt_step_cells(const ani_opt_state* state, const float* grad, const double* energies,
                            const float* lattice, float* coords, void* stream);
/*  Variable cell (ani_b200_opt_cell_step): FIRE on the degrees of freedom of ASE's FrechetCellFilter, every conformer  */
/*    fully periodic, over A + 3 rows: A atom rows u_i = F^-1 r_i (state->x holds u) and 3 cell rows d = c logm(F),     */
/*    where F is the deformation gradient (cell h = h0 F^T, rows are lattice vectors) and c = params[1].  Per conformer  */
/*    and step t, with W the force step's virial (its slots summed in a fixed order, Hartree), V = |det h|, L = d / c:  */
/*      atom rows   g_i = F^T f_i  (f = -dE/dr * force_scale, eV / A)                                                 */
/*      cell rows   Phi = D_expm(L^T)[G] / c,  G = -(W + p0 V I) F^-T * params[2]   (the Frechet derivative of expm at  */
/*                  L^T in the direction G: -dH/dd of the enthalpy H = E + p0 V, in eV with params[2] = HARTREE_TO_EV) */
/*                  projection 1: Phi -> (tr Phi / 3) I (hydrostatic strain);  2: Phi -> Phi - (tr Phi / 3) I          */
/*                  (constant volume)                                                                                */
/*    and then ani_b200_opt_step's FIRE over the A + 3 rows: P, F2, V2 and fmax include the cell rows, the maxstep      */
/*    clamp is over all of them, and a converged conformer freezes its cell too.  d(t+1) = d + s v_cell',               */
/*    F(t+1) = expm(d(t+1) / c), u(t+1) = u + s v'; the f32 coords of F(t+1) u(t+1) are wrapped into the               */
/*    float32-rounded h0 F(t+1)^T, which is also written to cell_out for the next force step (never read by this        */
/*    step).  Both exponentials run in float64 (Taylor series with scaling and squaring, ~1e-15 relative).             */
/*    ani_opt_cell (device pointers):                                                                                 */
/*      master      f64[2][n_conf][ANI_OPT_CELL_MASTER] {d, v_cell, F} (3 x 3 each, row-major) by step parity: step t   */
/*                  reads slot t % 2 and block 0 writes slot (t + 1) % 2 (v_cell too: every block of step t reads it)   */
/*      h0          f64[n_conf][9] the cell of construction (rows)                                                    */
/*      params      f64[n_conf][ANI_OPT_CELL_PARAMS] {p0 (Hartree / A^3), c (> 0), the unit of the cell forces per     */
/*                  Hartree (HARTREE_TO_EV, as force_scale)}                                                           */
/*      cell_out    f32 cell rows of conformer c at cell_out + c * cell_stride (>= 9): the workspace's cell, or its     */
/*                  cells of grid mode 3                                                                              */
/*      virial      f64[n_conf][virial_slots][9] the force step's virial slots                                         */
/*      cell_force  f64[n_conf][9] scratch: Phi of step t, written by the first launch, read by the second           */
/*      record      f64[record_rows][n_conf][ANI_OPT_CELL_RECORD] {V (A^3), -tr W / (3 V) (Hartree / A^3),            */
/*                  H = E + p0 V (Hartree)} of step t, in row t % record_rows, beside state->record                    */
/*      projection  0 none, 1 hydrostatic strain, 2 constant volume                                                   */
/*  ani_b200_opt_cell_init  one launch: with reset, v = 0, the scalars of slot counter[0] % 2 = {dt0, astart, 0} and    */
/*                     the master slot counter[0] % 2 = {0, 0, I}; then, from that slot's F, the f32 cell h0 F^T to     */
/*                     cell_out and the f32 coords of F u wrapped into it.                                            */
/*  ani_b200_opt_cell_step  after the force step at u(t), d(t) (grad, energies, and the virial slots): two launches,   */
/*                     the same two as ani_b200_opt_step.  Sums are float64 in a fixed order without atomics: the same  */
/*                     state and forces give the same bits.                                                           */
#define ANI_OPT_CELL_MASTER 27
#define ANI_OPT_CELL_PARAMS 3
#define ANI_OPT_CELL_RECORD 3
typedef struct ani_opt_cell {
  double* master;
  const double* h0;
  const double* params;
  float* cell_out;
  const double* virial;
  double* cell_force;
  double* record;
  int32_t cell_stride, virial_slots, projection, pad_;
} ani_opt_cell;
int ani_b200_opt_cell_init(const ani_opt_state* state, const ani_opt_cell* cell, int reset, float* coords,
                           void* stream);
int ani_b200_opt_cell_step(const ani_opt_state* state, const ani_opt_cell* cell, const float* grad,
                           const double* energies, float* coords, void* stream);
/*  L-BFGS (csrc/lbfgs.cu): ASE's ase.optimize.LBFGS without its line search, one independent optimisation per        */
/*    conformer, with the direction from the compact representation of the inverse BFGS matrix (Byrd, Nocedal &      */
/*    Schnabel, Math. Prog. 63 (1994)).  Units: A, eV, Hartree.  ani_lbfgs_state (device pointers; M = memory + 1):    */
/*      x, x_prev, g_prev  f64[n][3] positions (unwrapped, input order), those of the last step and its gradient       */
/*                  g = dE/dx * force_scale (eV / A)                                                                 */
/*      s, y        f64[n_conf][M][n_per_conf][3] ring of the pairs s = x(t) - x(t-1), y = g(t) - g(t-1): with head    */
/*                  the pairs ever stored and L = min(memory, head), chronological pair j is in slot (head - L + j) % M; */
/*                  the spare slot takes the next pair before it is known whether y.s == 0                           */
/*      sy, yy      f64[n_conf][M][M] slot-indexed s_i.y_j (for i not newer than j) and y_i.y_j                        */
/*      coef        f64[n_conf][2][memory] scratch: a and b of the step (chronological)                               */
/*      p           f64[n][3] scratch: the step's direction                                                          */
/*      iter        i64[n_conf][2] {k, head}: the steps taken (ASE's iteration) and the pairs ever stored              */
/*      force_scale f64[n] as in ani_opt_state                                                                        */
/*      params      f64[n_conf][ANI_LBFGS_PARAMS] per conformer: maxstep (A), damping, H0 = 1 / alpha (A^2 / eV), the  */
/*                  fmax threshold (eV / A); not read by the validation (device memory): the caller keeps them > 0     */
/*      counter, conv_step, record (ANI_LBFGS_RECORD = {t, E, fmax}) as in ani_opt_state                               */
/*      partials    f64[ANI_LBFGS_PARTIALS(n_conf, n_per_conf, memory)] scratch of ani_b200_lbfgs_step                  */
/*      memory      1 .. ANI_LBFGS_MAX_MEMORY (R of the solve, memory^2 doubles, sits in shared memory)                */
/*  ani_b200_lbfgs_init  with reset: x_prev = x, g_prev = 0, {k, head} = {0, 0}; then the f32 coords of x, wrapped     */
/*                     into the cell (cell_mode as ani_b200_opt_init).  One launch.                                   */
/*  ani_b200_lbfgs_step  after the force step at x(t) (grad f32[n][3] dE/dx, energies f64[n_conf]), four launches, per   */
/*                     conformer with fmax(t) = max_i |g_i|:                                                          */
/*                       record {t, E, fmax(t)};  fmax(t) < threshold (and running): conv_step = t, and from then on    */
/*                       nothing of the conformer changes;  else                                                      */
/*                       k >= 1: the pair s = x - x_prev, y = g - g_prev joins the history (the oldest leaves a full     */
/*                               one), unless y.s == 0, where it is skipped                                           */
/*                       p = -H g, H the inverse BFGS matrix of the live pairs with H0 (the two-loop recursion's p)     */
/*                       x(t+1) = x + damping p min(1, maxstep / max_i |p_i|)  (the factor applies when >= maxstep)   */
/*                       x_prev = x, g_prev = g, k += 1                                                               */
/*                     then the f32 coords of x(t+1) (wrapped into `cell` f32[9] when not NULL), and t += 1.  Sums are   */
/*                     float64 in a fixed order without atomics: the same state and forces give the same bits.          */
/*  ani_b200_lbfgs_step_cells  the same with one cell per conformer: the lattice table of grid mode 3                  */
/*                     (f32[n_conf][ANI_LATTICE_STRIDE], written by ani_b200_prepare_step_cells) in place of `cell`.    */
#define ANI_LBFGS_PARAMS 4
#define ANI_LBFGS_RECORD 3
#define ANI_LBFGS_MAX_MEMORY 128
#define ANI_LBFGS_TILE 32 /* atoms per tile of the dot sweep and per block of the direction launch */
#define ANI_LBFGS_PARTIALS(n_conf, n_per_conf, memory) \
  ((size_t)(n_conf) * (((n_per_conf) + ANI_LBFGS_TILE - 1) / ANI_LBFGS_TILE) * (4 * ((size_t)(memory) + 1) + 2))
typedef struct ani_lbfgs_state {
  double* x;
  double* x_prev;
  double* g_prev;
  double* s;
  double* y;
  double* sy;
  double* yy;
  double* coef;
  double* p;
  long long* iter;
  const double* force_scale;
  const double* params;
  long long* counter;
  long long* conv_step;
  double* record;
  double* partials;
  int32_t n_conf, n_per_conf, memory, record_rows;
} ani_lbfgs_state;
int ani_b200_lbfgs_init(const ani_lbfgs_state* state, const float* cells, int cell_mode, int reset, float* coords,
                        void* stream);
int ani_b200_lbfgs_step(const ani_lbfgs_state* state, const float* grad, const double* energies, const float* cell,
                        float* coords, void* stream);
int ani_b200_lbfgs_step_cells(const ani_lbfgs_state* state, const float* grad, const double* energies,
                              const float* lattice, float* coords, void* stream);
/*  Nudged elastic band (csrc/neb.cu): ASE's NEB ("aseneb" or "improvedtangent", optionally with a climbing image)     */
/*    relaxed by ASE's FIRE over each band's interior rows.  A band has n = n_images >= 3 images; images 0 and n - 1    */
/*    never move.  Interior image i (1 .. n - 2) of band b is conformer b (n - 2) + i - 1 of the force step, so the   */
/*    force step's flat atom index and the band's FIRE row index are the same.  Units: A, eV, Hartree.                 */
/*    ani_neb_state (device pointers):                                                                                */
/*      fire        the FIRE state of ani_opt_state with n_conf = B bands and n_per_conf = (n - 2) n_atoms rows: x, v,  */
/*                  force_scale, params (ANI_OPT_PARAMS per band), scalars, counter and conv_step as there; record      */
/*                  f64[record_rows][B][ANI_NEB_RECORD] {t, E_imax (Hartree), fmax (eV / A), imax}; partials           */
/*                  f64[B (n - 2)][ceil(n_atoms / ANI_MD_BLOCK)][4] scratch                                            */
/*      endpoints   f64[B][2][n_atoms][3] images 0 and n - 1                                                          */
/*      end_energies f64[B][2] their energies (Hartree)                                                               */
/*      springs     f64[B][n - 1] k_j (eV / A^2) of the spring between images j and j + 1                             */
/*      climb       f64[B] 1: image imax of the band climbs, 0: it does not                                           */
/*      neb_force   f64[B (n - 2) n_atoms][3] scratch: the NEB forces f (eV / A) of the step                          */
/*      dots        f64[B (n - 2)][ceil(n_atoms / ANI_MD_BLOCK)][ANI_NEB_DOTS] scratch                                 */
/*      method      ANI_NEB_ASENEB or ANI_NEB_IMPROVED_TANGENT                                                        */
/*    Per interior image i, with F = -dE/dx * force_scale, t- = x_i - x_{i-1}, t+ = x_{i+1} - x_i (both 0 where        */
/*    force_scale is 0), k- = k_{i-1}, k+ = k_i, imax = 1 + the first index of the largest of E_1 .. E_{n-2}, the       */
/*    tangent tau = alpha t- + beta t+ and f = F + gamma- t- + gamma+ t+:                                             */
/*      ASENEB       (alpha, beta) = (0, 1) for i < imax, (1, 0) for i > imax, (1, 1) at imax; m = tau.tau (1 if 0);  */
/*                   climbing: f = F - 2 (F.tau / m) tau;  else f = F - ((F.tau + (k- t- - k+ t+).tau) / m) tau        */
/*      IMPROVED_TANGENT  (Henkelman & Jonsson 2000) E_{i+1} > E_i > E_{i-1}: (0, 1);  E_{i+1} < E_i < E_{i-1}: (1, 0); */
/*                   else (dmin, dmax) if E_{i+1} > E_{i-1}, (dmax, dmin) if not, of |E_{i+1} - E_i|, |E_{i-1} - E_i|;  */
/*                   u = tau / |tau| (0 if |tau| = 0); climbing: f = F - 2 (F.u) u;                                  */
/*                   else f = F - (F.u) u + (k+ |t+| - k- |t-|) u                                                     */
/*    and then ani_b200_opt_step's FIRE per band over all its (n - 2) n_atoms rows (P, F2, V2, fmax and the maxstep     */
/*    clamp over the whole band; a converged band's x and v freeze).                                                  */
/*  ani_b200_neb_init  with reset: v = 0 and the scalars of slot counter[0] % 2 = {dt0, astart, 0}; then the f32       */
/*                     coords of x: cell_mode 0 open, 1 one cell f32[9], 2 one cell per force-step conformer            */
/*                     f32[B (n - 2)][9].  One launch.                                                                */
/*  ani_b200_neb_step  after the force step at x(t) (grad f32[B (n - 2) n_atoms][3] dE/dx, energies f64[B (n - 2)]),   */
/*                     three launches: the five dot products {t-.t-, t+.t+, t-.t+, F.t-, F.t+} per image, the NEB       */
/*                     forces and their FIRE partials, and FIRE's update; then the f32 coords of x(t+1) (wrapped into   */
/*                     `cell` f32[9] when not NULL), and t += 1.  Sums are float64 in a fixed order without atomics:    */
/*                     the same state and forces give the same bits.                                                 */
/*  ani_b200_neb_step_cells  the same with the lattice table of grid mode 3 (f32[B (n - 2)][ANI_LATTICE_STRIDE]) in    */
/*                     place of `cell`.                                                                              */
/*  ani_b200_neb_project  the first two launches only: neb_force of the current forces; writes nothing but scratch.    */
#define ANI_NEB_RECORD 4
#define ANI_NEB_DOTS 5
#define ANI_NEB_ASENEB 0
#define ANI_NEB_IMPROVED_TANGENT 1
typedef struct ani_neb_state {
  ani_opt_state fire;
  const double* endpoints;
  const double* end_energies;
  const double* springs;
  const double* climb;
  double* neb_force;
  double* dots;
  int32_t n_images, n_atoms, method, pad_;
} ani_neb_state;
int ani_b200_neb_init(const ani_neb_state* state, const float* cells, int cell_mode, int reset, float* coords,
                      void* stream);
int ani_b200_neb_step(const ani_neb_state* state, const float* grad, const double* energies, const float* cell,
                      float* coords, void* stream);
int ani_b200_neb_step_cells(const ani_neb_state* state, const float* grad, const double* energies,
                            const float* lattice, float* coords, void* stream);
int ani_b200_neb_project(const ani_neb_state* state, const float* grad, const double* energies, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ANI_B200_H */
