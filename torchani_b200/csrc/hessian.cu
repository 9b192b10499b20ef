// Analytic Hessians of open systems, after an ordinary step with gradients (include/ani_b200.h section 9).
//
// E = sum_i NN_s(i)(A_i) + pair terms, and A_i depends only on the vectors r_ij = x_j - x_i to i's neighbours within
// Rcr.  Per atom i the kernels build one block B_i over those relative vectors (3 n_i x 3 n_i, row / column 3 n + c =
// component c of neighbour n of the step's neighbour words):
//   network term    J_i^T K_i J_i with J_i = dA_i / dr_i. (ani_b200_hessian_jacobian writes its rows) and K_i the
//                   Hessian of the active members' weighted networks, formed as Zdot1^T Deltadot1 by a tangent pass
//                   over the rows (ani_b200_hessian_network): no K_i is ever stored
//   geometric term  the Hessian of g_i . A_i(r) with g_i = dE/dA_i (the step's dE/dAEV row) held fixed, plus the xTB /
//                   ZBL pair terms of the same neighbour list (ani_b200_hessian_geometric)
// and ani_b200_hessian_assemble maps B_i onto atoms {i} u nbrs(i) of the dense Hessian: (j, k) -> (j, k), (i, k) and
// (j, i) take -B, (i, i) takes the sum of B (translation invariance), accumulated in float64.
//
// Not the MD hot path: plain fp32 arithmetic with the accurate library functions (no MUFU approximations), no tensor
// cores, no operand pieces beyond reading the step's tiled AEVs.
#include <math.h>

#include "common.cuh"

namespace ani {

constexpr int HESS_TILE = ANI_HESSIAN_ROW_ALIGN;   // rows per GEMM row tile (one species each)

// ---- AEV pieces with first and second derivatives -------------------------------------------------------------------
// cutoff fc(R) and its first two derivatives (cutoffs.py:70-101); kind 0 cosine, 1 smooth(2, 1e-10), 2 none
__device__ __forceinline__ void cutoff_d2(float r, float rc, int kind, float& f, float& df, float& d2f) {
  if (kind == 2) {
    f = 1.f;
    df = d2f = 0.f;
  } else if (kind == 0) {
    const float a = 3.14159265358979323846f / rc;
    float s, c;
    sincospif(r / rc, &s, &c);
    f = 0.5f * c + 0.5f;
    df = -0.5f * a * s;
    d2f = -0.5f * a * a * c;
  } else {
    const float x = r / rc, u = 1.0f - x * x;
    if (u > 1e-10f) {
      f = expf(1.0f - 1.0f / u);
      const float g = -2.0f * x / (rc * u * u);   // d ln f / dR
      df = f * g;
      d2f = f * (g * g - 2.0f / (rc * rc) * (1.0f / (u * u) + 4.0f * x * x / (u * u * u)));
    } else {
      f = expf(1.0f - 1e10f);
      df = d2f = 0.f;
    }
  }
}

// angular factor F1(C) = ((1 + cos(acos(0.95 C) - ShfZ)) / 2)^zeta and its first two derivatives with respect to C
__device__ __forceinline__ void angular_f1(float C, float cz, float sz, float zeta, float& f, float& df, float& d2f) {
  const float c = 0.95f * C;
  const float s = sqrtf(fmaxf(1.0f - c * c, 1e-30f));
  const float b = fmaxf(0.5f + 0.5f * (c * cz + s * sz), 0.f);
  const float bc = 0.5f * (cz - c * sz / s);
  const float bcc = -0.5f * sz / (s * s * s);
  if (b <= 0.f) {
    f = df = d2f = 0.f;
    return;
  }
  const float p2 = powf(b, zeta - 2.0f);
  const float p1 = p2 * b;
  f = p1 * b;
  df = 0.95f * zeta * p1 * bc;
  d2f = 0.9025f * (zeta * (zeta - 1.0f) * p2 * bc * bc + zeta * p1 * bcc);
}

// r_j - r_i of the n-th neighbour word of sorted atom i (open systems: no image shifts), its length and species
__device__ __forceinline__ float4 neighbour_vector(const float4* __restrict__ spos, const int32_t* __restrict__ nbr_list,
                                                  int cap, int i, int n, int& sj) {
  const int j = nbr_list[(size_t)i * cap + n] & ANI_IDX_MASK;
  const float4 pi = spos[i], pj = spos[j];
  const float dx = pj.x - pi.x, dy = pj.y - pi.y, dz = pj.z - pi.z;
  sj = __float_as_int(pj.w);
  return make_float4(dx, dy, dz, sqrtf(dx * dx + dy * dy + dz * dz));
}

__device__ __forceinline__ int slot_count(const int32_t* __restrict__ nbr_cnt, int cap, int atom) {
  return min(nbr_cnt[atom], cap);
}

// ---- 1. Jacobian rows -------------------------------------------------------------------------------------------------
// One CTA per slot, one warp per neighbour n: rows row_off + 3 n + c receive dA_i / d(r_n)_c in the internal column
// order (the rows are zeroed by the entry point).  Radial: lane = shift, species block of n only.  Angular: lane =
// feature (ShfA major, ShfZ minor), one pass per angular partner k, column block of the pair (s_n, s_k).
constexpr int JAC_WARPS = 4;

__global__ void __launch_bounds__(JAC_WARPS * 32)
    k_hessian_jacobian(const __grid_constant__ ani_aev_params P, const float4* __restrict__ spos,
                       const int32_t* __restrict__ nbr_cnt, const int32_t* __restrict__ nbr_list, int cap,
                       const int32_t* __restrict__ atom_of, const int32_t* __restrict__ row_off,
                       float* __restrict__ jac, int ldx) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int slot = blockIdx.x;
  const int i = atom_of[slot];
  const int cnt = slot_count(nbr_cnt, cap, i);
  const int nR = P.n_shf_r, RL = P.num_species * nR, NZ = P.n_shf_z;
  const int a_idx = lane / NZ, z_idx = lane % NZ;
  const float shf_a = P.shf_a[a_idx], cz = P.cos_z[z_idx], sz = P.sin_z[z_idx];
  for (int n = warp; n < cnt; n += JAC_WARPS) {
    int sn;
    const float4 d = neighbour_vector(spos, nbr_list, cap, i, n, sn);
    float* row = jac + (size_t)(row_off[slot] + 3 * n) * ldx;
    const float inv_r = 1.0f / d.w;
    const float ux = d.x * inv_r, uy = d.y * inv_r, uz = d.z * inv_r;
    if (lane < nR) {
      float fc, dfc, d2fc;
      cutoff_d2(d.w, P.rcr, P.cutoff_kind, fc, dfc, d2fc);
      const float x = d.w - P.shf_r[lane];
      const float G = 0.25f * expf(-P.eta_r * x * x);
      const float dv = G * (-2.0f * P.eta_r * x * fc + dfc);
      const int col = sn * nR + lane;
      row[col] = dv * ux;
      row[ldx + col] = dv * uy;
      row[2 * ldx + col] = dv * uz;
    }
    if (d.w > P.rca) continue;
    float fcn, dfcn, d2fcn;
    cutoff_d2(d.w, P.rca, P.cutoff_kind, fcn, dfcn, d2fcn);
    for (int k = 0; k < cnt; ++k) {
      if (k == n) continue;
      int sk;
      const float4 e = neighbour_vector(spos, nbr_list, cap, i, k, sk);
      if (e.w > P.rca) continue;
      float fck, dfck, d2fck;
      cutoff_d2(e.w, P.rca, P.cutoff_kind, fck, dfck, d2fck);
      const float inv_rr = 1.0f / fmaxf(d.w * e.w, 1e-10f);
      const float C = (d.x * e.x + d.y * e.y + d.z * e.z) * inv_rr;
      float f1, df1, d2f1;
      angular_f1(C, cz, sz, P.zeta, f1, df1, d2f1);
      const float q = 0.5f * (d.w + e.w) - shf_a;
      const float f2 = expf(-P.eta_a * q * q);
      const float df2 = -2.0f * P.eta_a * q * f2;   // d/dRbar; dRbar/dR_n = 1/2
      const float dT_dR = 2.0f * f1 * (0.5f * df2 * fcn * fck + f2 * dfcn * fck);
      const float dT_dC = 2.0f * df1 * f2 * fcn * fck;
      // dC/dr_n = r_k / (R_n R_k) - C r_n / R_n^2
      const float gx = dT_dR * ux + dT_dC * (e.x * inv_rr - C * ux * inv_r);
      const float gy = dT_dR * uy + dT_dC * (e.y * inv_rr - C * uy * inv_r);
      const float gz = dT_dR * uz + dT_dC * (e.z * inv_rr - C * uz * inv_r);
      const int col = RL + P.ang_pad + pair_index(sn, sk, P.num_species) * 32 + lane;
      row[col] += gx;
      row[ldx + col] += gy;
      row[2 * ldx + col] += gz;
    }
  }
}

// ---- 2. tangent network pass --------------------------------------------------------------------------------------------
// Per-slot primal vectors of one member, VEC_* x hmax floats each: sigma'(z1), sigma''(z1) (W2^T delta2),
// sigma'(z2), sigma''(z2) (W3^T delta3), w4 sigma''(z3)
enum { VEC_S1 = 0, VEC_R1 = 1, VEC_S2 = 2, VEC_R2 = 3, VEC_Q3 = 4, VEC_COUNT = 5 };

__device__ __forceinline__ void activation_d(int act, float alpha, float z, float& y, float& d1, float& d2) {
  if (act == ANI_ACT_CELU) {
    // CELU: at z = 0 both branches give y = 0 and sigma' = 1; sigma'' takes the linear branch's 0 there, as torch's
    // double backward does (its second derivative is non-zero for z < 0 only)
    if (z >= 0.f) {
      y = z;
      d1 = 1.f;
      d2 = 0.f;
    } else {
      const float e = expf(z / alpha);
      y = alpha * (e - 1.f);
      d1 = e;
      d2 = e / alpha;
    }
  } else {
    const float phi = 0.3989422804014327f * expf(-0.5f * z * z);
    const float Phi = 0.5f * erfcf(-z * 0.7071067811865476f);
    y = z * Phi;
    d1 = Phi + z * phi;
    d2 = phi * (2.0f - z * z);
  }
}

// one value of the step's tiled AEV operand
__device__ __forceinline__ float tiled_value(const unsigned char* __restrict__ x, int row, int col, int kblocks) {
  const unsigned char* p = x + opnd_offset(row, col, kblocks);
  float v = 0.f;
#pragma unroll
  for (int k = OPND_PARTS - 1; k >= 0; --k) {
    const unsigned short h = *reinterpret_cast<const unsigned short*>(p + k * OPND_PART_BYTES);
#if ANI_OPND_FP16X2
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(h));
    v += f;
#else
    v += __uint_as_float((uint32_t)h << 16);
#endif
  }
  return v / OPND_SCALE_VALUE;
}

// y[o] = b[o] + sum_k W[o][k] x[k] (W [no][ld]) or, transposed, y[o] = sum_k W[k][o] x[k] (W [nk][ld]); by the CTA
__device__ __forceinline__ void cta_matvec(const float* __restrict__ W, int ld, bool trans, int no, int nk,
                                           const float* x, const float* __restrict__ b, float* y) {
  for (int o = threadIdx.x; o < no; o += blockDim.x) {
    float acc = b ? b[o] : 0.f;
    if (trans)
      for (int k = 0; k < nk; ++k) acc = fmaf(W[(size_t)k * ld + o], x[k], acc);
    else
      for (int k = 0; k < nk; ++k) acc = fmaf(W[(size_t)o * ld + k], x[k], acc);
    y[o] = acc;
  }
  __syncthreads();
}

// One CTA per slot: the primal forward and backward of member m on the slot's AEV row, in fp32.
__global__ void k_hessian_primal(const __grid_constant__ ani_mlp_model M, const __grid_constant__ ani_hessian_weights W,
                                 int member, const unsigned char* __restrict__ x, const int32_t* __restrict__ row_of,
                                 const int32_t* __restrict__ atom_of, const float4* __restrict__ spos,
                                 float* __restrict__ vec, int hmax) {
  extern __shared__ float sm[];
  const int slot = blockIdx.x;
  const int i = atom_of[slot];
  const int s = __float_as_int(spos[i].w);
  const ani_mlp_species& sp = M.sp[s];
  const int h1 = sp.h1, h2 = sp.h2, h3 = sp.h3, ldx = M.ldx;
  float* a = sm;                 // [ldx]
  float* z1 = a + ldx;           // [hmax] each below
  float* y1 = z1 + hmax;
  float* z2 = y1 + hmax;
  float* y2 = z2 + hmax;
  float* z3 = y2 + hmax;
  float* t = z3 + hmax;
  float* e = t + hmax;
  const int row = row_of[i];
  for (int c = threadIdx.x; c < ldx; c += blockDim.x) a[c] = tiled_value(x, row, c, ldx >> 5);
  __syncthreads();
  const float* w1 = W.w1[s] + (size_t)member * h1 * ldx;
  const float* w2 = W.w2[s] + (size_t)member * h2 * h1;
  const float* w3 = W.w3[s] + (size_t)member * h3 * h2;
  const float* w4 = sp.w4 + (size_t)member * h3;
  float* v = vec + (size_t)slot * VEC_COUNT * hmax;
  const int act = M.activation;
  const float alpha = M.celu_alpha;
  float dd1, dd2;
  cta_matvec(w1, ldx, false, h1, ldx, a, sp.b1 + (size_t)member * h1, z1);
  for (int o = threadIdx.x; o < h1; o += blockDim.x) activation_d(act, alpha, z1[o], y1[o], dd1, dd2);
  __syncthreads();
  cta_matvec(w2, h1, false, h2, h1, y1, sp.b2 + (size_t)member * h2, z2);
  for (int o = threadIdx.x; o < h2; o += blockDim.x) activation_d(act, alpha, z2[o], y2[o], dd1, dd2);
  __syncthreads();
  cta_matvec(w3, h2, false, h3, h2, y2, sp.b3 + (size_t)member * h3, z3);
  // delta3 = w4 sigma'(z3); q3 = w4 sigma''(z3)
  for (int o = threadIdx.x; o < h3; o += blockDim.x) {
    float y;
    activation_d(act, alpha, z3[o], y, dd1, dd2);
    t[o] = w4[o] * dd1;
    v[VEC_Q3 * hmax + o] = w4[o] * dd2;
  }
  __syncthreads();
  cta_matvec(w3, h2, true, h2, h3, t, nullptr, e);   // e = W3^T delta3
  for (int o = threadIdx.x; o < h2; o += blockDim.x) {
    float y;
    activation_d(act, alpha, z2[o], y, dd1, dd2);
    v[VEC_S2 * hmax + o] = dd1;
    v[VEC_R2 * hmax + o] = dd2 * e[o];
    t[o] = dd1 * e[o];                               // delta2
  }
  __syncthreads();
  cta_matvec(w2, h1, true, h1, h2, t, nullptr, e);   // e = W2^T delta2
  for (int o = threadIdx.x; o < h1; o += blockDim.x) {
    float y;
    activation_d(act, alpha, z1[o], y, dd1, dd2);
    v[VEC_S1 * hmax + o] = dd1;
    v[VEC_R1 * hmax + o] = dd2 * e[o];
  }
}

// One layer of the tangent pass over the rows of a chunk: acc = A B^T with B[n][k] = W[n][k] (or W[k][n], TRANS_B), per
// 64-row tile of one species, then the epilogue
//   EPI_TANGENT  out0 = acc, out1 = vec[VA] * acc            (Zdot and sigma' Zdot of layers 1, 2)
//   EPI_SCALE    out0 = vec[VA] * acc                        (Deltadot3 = w4 sigma''(z3) Zdot3)
//   EPI_DELTA    out0 = vec[VA] * acc + vec[VB] * in         (Deltadot2, Deltadot1)
// with vec the slot's primal vectors; padding rows (row_slot < 0) get zeros.
enum { EPI_TANGENT = 0, EPI_SCALE = 1, EPI_DELTA = 2 };
constexpr int G_BM = 64, G_BN = 64, G_BK = 16;

struct TangentLayer {
  const float* b[ANI_MAX_SPECIES];
  int n[ANI_MAX_SPECIES], k[ANI_MAX_SPECIES], ldb[ANI_MAX_SPECIES];
};

template <bool TRANS_B, int EPI>
__global__ void __launch_bounds__(256)
    k_hessian_tangent_gemm(const __grid_constant__ TangentLayer L, const float* __restrict__ A, int lda,
                           const int32_t* __restrict__ tile_species, const int32_t* __restrict__ row_slot,
                           const float* __restrict__ vec, int hmax, int va, int vb, const float* __restrict__ in,
                           float* __restrict__ out0, float* __restrict__ out1, int ldo) {
  __shared__ float As[G_BK][G_BM + 4];
  __shared__ float Bs[G_BK][G_BN + 4];
  const int s = tile_species[blockIdx.y];
  const int N = L.n[s], K = L.k[s], ldb = L.ldb[s];
  const int n0 = blockIdx.x * G_BN, r0 = blockIdx.y * G_BM;
  if (n0 >= N) return;
  const float* __restrict__ B = L.b[s];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += G_BK) {
    for (int e = threadIdx.x; e < G_BM * G_BK; e += 256) {
      const int r = e / G_BK, kk = e % G_BK;
      As[kk][r] = A[(size_t)(r0 + r) * lda + k0 + kk];
      const int n = n0 + r;
      float bv = 0.f;
      if (n < N) bv = TRANS_B ? B[(size_t)(k0 + kk) * ldb + n] : B[(size_t)n * ldb + k0 + kk];
      Bs[kk][r] = bv;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < G_BK; ++kk) {
      float av[4], bv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        av[u] = As[kk][ty + 16 * u];
        bv[u] = Bs[kk][tx + 16 * u];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int w = 0; w < 4; ++w) acc[u][w] = fmaf(av[u], bv[w], acc[u][w]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int r = r0 + ty + 16 * u;
    const int slot = row_slot[r];
    const float* v = vec + (size_t)max(slot, 0) * VEC_COUNT * hmax;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const int n = n0 + tx + 16 * w;
      if (n >= N) continue;
      const size_t o = (size_t)r * ldo + n;
      const float x = acc[u][w];
      if (slot < 0) {
        out0[o] = 0.f;
        if (EPI == EPI_TANGENT) out1[o] = 0.f;
      } else if (EPI == EPI_TANGENT) {
        out0[o] = x;
        out1[o] = v[va * hmax + n] * x;
      } else if (EPI == EPI_SCALE) {
        out0[o] = v[va * hmax + n] * x;
      } else {
        out0[o] = fmaf(v[va * hmax + n], x, v[vb * hmax + n] * in[o]);
      }
    }
  }
}

// B_i += scale Zdot1_i Deltadot1_i^T over the slot's 3 n_i rows: one CTA per (slot, 32 x 32 output tile)
__global__ void __launch_bounds__(256)
    k_hessian_block_contract(const float* __restrict__ zd, const float* __restrict__ dd, int ld,
                             const int32_t* __restrict__ nbr_cnt, int cap, const int32_t* __restrict__ atom_of,
                             const int32_t* __restrict__ row_off, const long long* __restrict__ block_off,
                             const float4* __restrict__ spos, const __grid_constant__ ani_mlp_model M, float scale,
                             float* __restrict__ blocks) {
  __shared__ float Zs[32][33], Ds[32][33];
  const int slot = blockIdx.x;
  const int i = atom_of[slot];
  const int m3 = 3 * slot_count(nbr_cnt, cap, i);
  const int tiles = (m3 + 31) / 32;
  if ((int)blockIdx.y >= tiles * tiles) return;
  const int p0 = (blockIdx.y / tiles) * 32, q0 = (blockIdx.y % tiles) * 32;
  const int K = M.sp[__float_as_int(spos[i].w)].h1;
  const size_t rb = row_off[slot];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  float acc[2][2] = {};
  for (int k0 = 0; k0 < K; k0 += 32) {
    for (int e = threadIdx.x; e < 32 * 32; e += 256) {
      const int r = e / 32, kk = e % 32;
      Zs[r][kk] = p0 + r < m3 ? zd[(rb + p0 + r) * ld + k0 + kk] : 0.f;
      Ds[r][kk] = q0 + r < m3 ? dd[(rb + q0 + r) * ld + k0 + kk] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < 32; ++kk)
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int w = 0; w < 2; ++w) acc[u][w] = fmaf(Zs[ty + 16 * u][kk], Ds[tx + 16 * w][kk], acc[u][w]);
    __syncthreads();
  }
  float* B = blocks + block_off[slot];
#pragma unroll
  for (int u = 0; u < 2; ++u)
#pragma unroll
    for (int w = 0; w < 2; ++w) {
      const int p = p0 + ty + 16 * u, q = q0 + tx + 16 * w;
      if (p < m3 && q < m3) B[(size_t)p * m3 + q] += scale * acc[u][w];
    }
}

// ---- 3. geometric term ----------------------------------------------------------------------------------------------
// add a * u u^T + b * I into the 3 x 3 block (p, q) of B (rows 3p.., columns 3q..)
__device__ __forceinline__ void add_radial_block(float* B, int m3, int n, float a, float b, float ux, float uy,
                                                 float uz) {
  const float u[3] = {ux, uy, uz};
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int d = 0; d < 3; ++d) atomicAdd(&B[(size_t)(3 * n + c) * m3 + 3 * n + d], a * u[c] * u[d] + (c == d ? b : 0.f));
}

// second derivative of E(R) fc(R) of one pair potential (kinds 0 xTB, 1 ZBL) with respect to R, and the first
__device__ __forceinline__ void pair_d2(const ani_pair_params& P, int a, int b, float R, float& e1, float& e2) {
  const float tb = P.to_bohr;
  const float d = fmaxf(R, 1e-7f) * tb;
  float E, Ed, Edd;   // derivatives with respect to d
  if (P.kind == 0) {
    const float y = P.a[a][b], sa = P.b[a][b], k = P.c[a][b];
    const float dk = powf(d, k);
    E = y / d * expf(-sa * dk);
    const float Lg = -sa * k * dk / d - 1.0f / d;                    // d ln E / dd
    const float Lgd = -sa * k * (k - 1.0f) * dk / (d * d) + 1.0f / (d * d);
    Ed = E * Lg;
    Edd = E * (Lg * Lg + Lgd);
  } else {
    const float zz = P.a[a][b], s = P.b[a][b];
    float S = 0.f, Sd = 0.f, Sdd = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float x = P.screen_exp[q] * s;
      const float t = P.screen_coeff[q] * expf(-x * d);
      S += t;
      Sd -= x * t;
      Sdd += x * x * t;
    }
    E = zz * S / d;
    Ed = zz * (Sd / d - S / (d * d));
    Edd = zz * (Sdd / d - 2.0f * Sd / (d * d) + 2.0f * S / (d * d * d));
  }
  if (R < 1e-7f) Ed = Edd = 0.f;   // the clamp has no slope below its floor
  float f, df, d2f;
  cutoff_d2(R, P.cutoff, P.cutoff_fn, f, df, d2f);
  e1 = tb * Ed * f + E * df;
  e2 = tb * tb * Edd * f + 2.0f * tb * Ed * df + E * d2f;
}

// One CTA per slot.  With g (the step's dE/dAEV rows): radial blocks per neighbour, angular 6 x 6 blocks per pair of
// angular neighbours.  With a pair potential: its 1/2 E(R) fc(R) per neighbour within its cutoff (the step's atomic
// split of a full list).  Float atomics into B (blocks of one slot are shared by its threads).
__global__ void __launch_bounds__(128)
    k_hessian_geometric(const __grid_constant__ ani_aev_params P, const float4* __restrict__ spos,
                        const int32_t* __restrict__ nbr_cnt, const int32_t* __restrict__ nbr_list, int cap,
                        const int32_t* __restrict__ row_of, const float* __restrict__ g_all, int ldx,
                        const ani_pair_params* __restrict__ pair, const int32_t* __restrict__ atom_of,
                        const long long* __restrict__ block_off, float* __restrict__ blocks) {
  __shared__ float4 nd[256];
  __shared__ int nsp[256];
  __shared__ unsigned char aidx[256];
  __shared__ int n_ang;
  const int slot = blockIdx.x;
  const int i = atom_of[slot];
  const int cnt = slot_count(nbr_cnt, cap, i);
  const int m3 = 3 * cnt;
  const int si = __float_as_int(spos[i].w);
  float* B = blocks + block_off[slot];
  for (int n = threadIdx.x; n < cnt; n += blockDim.x) nd[n] = neighbour_vector(spos, nbr_list, cap, i, n, nsp[n]);
  __syncthreads();
  if (pair) {
    const ani_pair_params& pp = *pair;
    for (int n = threadIdx.x; n < cnt; n += blockDim.x) {
      const float4 d = nd[n];
      if (pp.cutoff_fn != 2 && d.w > pp.cutoff) continue;
      float e1, e2;
      pair_d2(pp, si, nsp[n], d.w, e1, e2);
      const float inv_r = 1.0f / d.w;
      add_radial_block(B, m3, n, 0.5f * (e2 - e1 * inv_r), 0.5f * e1 * inv_r, d.x * inv_r, d.y * inv_r, d.z * inv_r);
    }
    return;
  }
  const float* g = g_all + (size_t)row_of[i] * ldx;
  const int nR = P.n_shf_r, RL = P.num_species * nR, NA = P.n_shf_a, NZ = P.n_shf_z;
  // radial: f(R) = sum_m g_m 0.25 exp(-eta (R - ShfR_m)^2) fc(R)
  for (int n = threadIdx.x; n < cnt; n += blockDim.x) {
    const float4 d = nd[n];
    float fc, dfc, d2fc;
    cutoff_d2(d.w, P.rcr, P.cutoff_kind, fc, dfc, d2fc);
    float f1 = 0.f, f2 = 0.f;
    for (int m = 0; m < nR; ++m) {
      const float x = d.w - P.shf_r[m];
      const float G = 0.25f * expf(-P.eta_r * x * x);
      const float Gd = -2.0f * P.eta_r * x * G;
      const float Gdd = (4.0f * P.eta_r * P.eta_r * x * x - 2.0f * P.eta_r) * G;
      const float gm = g[nsp[n] * nR + m];
      f1 = fmaf(gm, Gd * fc + G * dfc, f1);
      f2 = fmaf(gm, Gdd * fc + 2.0f * Gd * dfc + G * d2fc, f2);
    }
    const float inv_r = 1.0f / d.w;
    add_radial_block(B, m3, n, f2 - f1 * inv_r, f1 * inv_r, d.x * inv_r, d.y * inv_r, d.z * inv_r);
  }
  if (threadIdx.x == 0) {
    int c = 0;
    for (int n = 0; n < cnt; ++n)
      if (nd[n].w <= P.rca && c < ANI_MAX_ANG) aidx[c++] = (unsigned char)n;
    n_ang = c;
  }
  __syncthreads();
  const int na = n_ang;
  const int pairs = na * (na - 1) / 2;
  for (int t = threadIdx.x; t < pairs; t += blockDim.x) {
    // t-th pair (ja < jb) of the triangle
    int jb = (int)(0.5f + 0.5f * sqrtf(1.0f + 8.0f * (float)t));
    while (jb * (jb - 1) / 2 > t) --jb;
    while ((jb + 1) * jb / 2 <= t) ++jb;
    const int ja = t - jb * (jb - 1) / 2;
    const int n = aidx[ja], k = aidx[jb];
    const float4 a4 = nd[n], b4 = nd[k];
    const float A = a4.w, Bl = b4.w;
    const float ua[3] = {a4.x / A, a4.y / A, a4.z / A}, ub[3] = {b4.x / Bl, b4.y / Bl, b4.z / Bl};
    const float C = (a4.x * b4.x + a4.y * b4.y + a4.z * b4.z) / fmaxf(A * Bl, 1e-10f);
    const float* gp = g + RL + P.ang_pad + pair_index(nsp[n], nsp[k], P.num_species) * 32;
    // S_uv = sum g F1^(u) F2^(v) (derivatives of F1 in C, of F2 in Rbar)
    float S00 = 0.f, S10 = 0.f, S20 = 0.f, S01 = 0.f, S02 = 0.f, S11 = 0.f;
    const float rbar = 0.5f * (A + Bl);
    for (int z = 0; z < NZ; ++z) {
      float f1, df1, d2f1;
      angular_f1(C, P.cos_z[z], P.sin_z[z], P.zeta, f1, df1, d2f1);
      float t0 = 0.f, t1 = 0.f, t2 = 0.f;
      for (int aa = 0; aa < NA; ++aa) {
        const float q = rbar - P.shf_a[aa];
        const float f2 = expf(-P.eta_a * q * q);
        const float gv = gp[aa * NZ + z];
        t0 = fmaf(gv, f2, t0);
        t1 = fmaf(gv, -2.0f * P.eta_a * q * f2, t1);
        t2 = fmaf(gv, (4.0f * P.eta_a * P.eta_a * q * q - 2.0f * P.eta_a) * f2, t2);
      }
      S00 = fmaf(f1, t0, S00);
      S10 = fmaf(df1, t0, S10);
      S20 = fmaf(d2f1, t0, S20);
      S01 = fmaf(f1, t1, S01);
      S02 = fmaf(f1, t2, S02);
      S11 = fmaf(df1, t1, S11);
    }
    float fa, dfa, d2fa, fb, dfb, d2fb;
    cutoff_d2(A, P.rca, P.cutoff_kind, fa, dfa, d2fa);
    cutoff_d2(Bl, P.rca, P.cutoff_kind, fb, dfb, d2fb);
    const float W = fa * fb;
    // phi(A, B, C) = 2 fc(A) fc(B) sum g F1(C) F2((A + B) / 2)
    const float pA = 2.0f * (dfa * fb * S00 + 0.5f * W * S01);
    const float pB = 2.0f * (fa * dfb * S00 + 0.5f * W * S01);
    const float pC = 2.0f * W * S10;
    const float pAA = 2.0f * (d2fa * fb * S00 + dfa * fb * S01 + 0.25f * W * S02);
    const float pBB = 2.0f * (fa * d2fb * S00 + fa * dfb * S01 + 0.25f * W * S02);
    const float pAB = 2.0f * (dfa * dfb * S00 + 0.5f * (dfa * fb + fa * dfb) * S01 + 0.25f * W * S02);
    const float pAC = 2.0f * (dfa * fb * S10 + 0.5f * W * S11);
    const float pBC = 2.0f * (fa * dfb * S10 + 0.5f * W * S11);
    const float pCC = 2.0f * W * S20;
    float gA[3], gB[3];   // dC/dr_a, dC/dr_b
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      gA[c] = (ub[c] - C * ua[c]) / A;
      gB[c] = (ua[c] - C * ub[c]) / Bl;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        const float id = c == d ? 1.f : 0.f;
        const float haa = pAA * ua[c] * ua[d] + pCC * gA[c] * gA[d] + pAC * (ua[c] * gA[d] + gA[c] * ua[d]) +
                          pA * (id - ua[c] * ua[d]) / A +
                          pC * (-(gA[c] * ua[d] + ua[c] * gA[d]) / A + C * (ua[c] * ua[d] - id) / (A * A));
        const float hbb = pBB * ub[c] * ub[d] + pCC * gB[c] * gB[d] + pBC * (ub[c] * gB[d] + gB[c] * ub[d]) +
                          pB * (id - ub[c] * ub[d]) / Bl +
                          pC * (-(gB[c] * ub[d] + ub[c] * gB[d]) / Bl + C * (ub[c] * ub[d] - id) / (Bl * Bl));
        const float hab = pAB * ua[c] * ub[d] + pCC * gA[c] * gB[d] + pAC * ua[c] * gB[d] + pBC * gA[c] * ub[d] +
                          pC * (id - ub[c] * ub[d] - ua[c] * ua[d] + C * ua[c] * ub[d]) / (A * Bl);
        atomicAdd(&B[(size_t)(3 * n + c) * m3 + 3 * n + d], haa);
        atomicAdd(&B[(size_t)(3 * k + c) * m3 + 3 * k + d], hbb);
        atomicAdd(&B[(size_t)(3 * n + c) * m3 + 3 * k + d], hab);
        atomicAdd(&B[(size_t)(3 * k + d) * m3 + 3 * n + c], hab);
      }
  }
}

// ---- 4. assembly ------------------------------------------------------------------------------------------------------
// One CTA per slot: B_i through P_i into hess (float64, [n_conf][3 A][3 A], input atom order).
__global__ void __launch_bounds__(256)
    k_hessian_assemble(const int32_t* __restrict__ nbr_cnt, const int32_t* __restrict__ nbr_list, int cap,
                       const int32_t* __restrict__ sorted_orig, const int32_t* __restrict__ atom_of,
                       const long long* __restrict__ block_off, const float* __restrict__ blocks, int n_per_conf,
                       double* __restrict__ hess) {
  __shared__ int col[768];
  __shared__ double total[9];
  const int slot = blockIdx.x;
  const int i = atom_of[slot];
  const int cnt = slot_count(nbr_cnt, cap, i);
  const int m3 = 3 * cnt;
  const int oi = sorted_orig[i];
  const int conf = oi / n_per_conf;
  const size_t D = 3 * (size_t)n_per_conf;
  double* H = hess + (size_t)conf * D * D;
  const int ci = 3 * (oi - conf * n_per_conf);
  const float* B = blocks + block_off[slot];
  for (int p = threadIdx.x; p < m3; p += blockDim.x) {
    const int j = nbr_list[(size_t)i * cap + p / 3] & ANI_IDX_MASK;
    col[p] = 3 * (sorted_orig[j] - conf * n_per_conf) + p % 3;
  }
  if (threadIdx.x < 9) total[threadIdx.x] = 0.0;
  __syncthreads();
  for (size_t e = threadIdx.x; e < (size_t)m3 * m3; e += blockDim.x) {
    const int p = (int)(e / m3), q = (int)(e % m3);
    atomicAdd(&H[(size_t)col[p] * D + col[q]], (double)B[e]);
  }
  // (i, k) takes minus the column sums over the neighbours j, (j, i) minus the row sums, (i, i) the total
  for (int q = threadIdx.x; q < m3; q += blockDim.x) {
    double cs[3] = {0.0, 0.0, 0.0}, rs[3] = {0.0, 0.0, 0.0};
    for (int p = 0; p < m3; p += 3) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        cs[c] += (double)B[(size_t)(p + c) * m3 + q];
        rs[c] += (double)B[(size_t)q * m3 + p + c];
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      atomicAdd(&H[(size_t)(ci + c) * D + col[q]], -cs[c]);
      atomicAdd(&H[(size_t)col[q] * D + ci + c], -rs[c]);
      atomicAdd(&total[(q % 3) * 3 + c], rs[c]);
    }
  }
  __syncthreads();
  if (threadIdx.x < 9) atomicAdd(&H[(size_t)(ci + threadIdx.x / 3) * D + ci + threadIdx.x % 3], total[threadIdx.x]);
}

static int check_chunk(const ani_hessian_chunk* ch) {
  if (!ch || !ch->atom || !ch->row_off || !ch->block_off || ch->n_slots < 0) return ANI_ERR_BAD_ARG;
  if (ch->rows < 0 || ch->rows % HESS_TILE || ch->max_count < 0) return ANI_ERR_BAD_ARG;
  return ANI_OK;
}

}  // namespace ani

using namespace ani;

extern "C" int ani_b200_hessian_jacobian(const ani_aev_params* params, const float* spos, const int32_t* nbr_cnt,
                                         const int32_t* nbr_list, int cap, const ani_hessian_chunk* chunk, float* jac,
                                         int ldx, void* stream) {
  if (!params || !spos || !nbr_cnt || !nbr_list || !jac || cap < 1 || cap > 256 || ldx % 32) return ANI_ERR_BAD_ARG;
  if (int rc = check_chunk(chunk)) return rc;
  if (params->n_shf_a * params->n_shf_z != 32 || params->n_shf_r > 32) return ANI_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaMemsetAsync(jac, 0, (size_t)chunk->rows * ldx * sizeof(float), st) != cudaSuccess) {
    set_cuda_error(cudaGetLastError());
    return ANI_ERR_CUDA;
  }
  if (chunk->n_slots == 0) return ANI_OK;
  k_hessian_jacobian<<<chunk->n_slots, JAC_WARPS * 32, 0, st>>>(*params, reinterpret_cast<const float4*>(spos),
                                                                   nbr_cnt, nbr_list, cap, chunk->atom, chunk->row_off,
                                                                   jac, ldx);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_hessian_network(const ani_mlp_model* model, const ani_hessian_weights* weights, const void* x,
                                        const int32_t* row_of, const float* spos, const int32_t* nbr_cnt, int cap,
                                        const ani_hessian_chunk* chunk, const float* jac, float* scratch,
                                        float* blocks, void* stream) {
  if (!model || !weights || !x || !row_of || !spos || !nbr_cnt || !jac || !scratch || !blocks || cap < 1 || cap > 256)
    return ANI_ERR_BAD_ARG;
  if (int rc = check_chunk(chunk)) return rc;
  if (!chunk->row_slot || !chunk->tile_species) return ANI_ERR_BAD_ARG;
  if (model->activation != ANI_ACT_CELU && model->activation != ANI_ACT_GELU) return ANI_ERR_BAD_ARG;
  const int S = model->num_species, ldx = model->ldx;
  if (S < 1 || S > ANI_MAX_SPECIES || model->num_members < 1 || model->num_members > ANI_MAX_MEMBERS || ldx % 32)
    return ANI_ERR_BAD_ARG;
  for (int s = 0; s < S; ++s)
    if (!weights->w1[s] || !weights->w2[s] || !weights->w3[s]) return ANI_ERR_BAD_ARG;
  if (chunk->n_slots == 0) return ANI_OK;
  const int hmax = ani_b200_hessian_hidden_max(model);
  const size_t R = chunk->rows;
  float* zd1 = scratch;                 // Zdot1, kept to the contraction
  float* zd2 = zd1 + R * hmax;          // Zdot2, kept to Deltadot2
  float* u = zd2 + R * hmax;            // sigma'(z1) Zdot1, then Deltadot3, then Deltadot1
  float* v = u + R * hmax;              // sigma'(z2) Zdot2, then Deltadot2
  float* vec = v + R * hmax;            // [n_slots][VEC_COUNT][hmax]
  cudaStream_t st = (cudaStream_t)stream;
  const int sps = 256;
  const size_t primal_smem = (size_t)(ldx + 7 * hmax) * sizeof(float);
  if (primal_smem > 48 * 1024 &&
      cudaFuncSetAttribute(k_hessian_primal, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)primal_smem) !=
          cudaSuccess) {
    set_cuda_error(cudaGetLastError());
    return ANI_ERR_CUDA;
  }
  const dim3 grid_g((hmax + G_BN - 1) / G_BN, chunk->rows / G_BM);
  const int tiles = (3 * min(chunk->max_count, cap) + 31) / 32;
  if (tiles == 0) return ANI_OK;   // no atom of the chunk has a neighbour: every B_i is empty (and a 0-tile grid invalid)
  const float4* sp4 = reinterpret_cast<const float4*>(spos);
  for (int m = 0; m < model->num_members; ++m) {
    const float scale = model->member_scale[m];
    if (scale == 0.f) continue;
    k_hessian_primal<<<chunk->n_slots, sps, primal_smem, st>>>(*model, *weights, m,
                                                               reinterpret_cast<const unsigned char*>(x), row_of,
                                                               chunk->atom, sp4, vec, hmax);
    ANI_CUDA_CHECK_LAUNCH();
    TangentLayer l1{}, l2{}, l3{}, l3t{}, l2t{};
    for (int s = 0; s < S; ++s) {
      const ani_mlp_species& q = model->sp[s];
      l1.b[s] = weights->w1[s] + (size_t)m * q.h1 * ldx;
      l1.n[s] = q.h1, l1.k[s] = ldx, l1.ldb[s] = ldx;
      l2.b[s] = weights->w2[s] + (size_t)m * q.h2 * q.h1;
      l2.n[s] = q.h2, l2.k[s] = q.h1, l2.ldb[s] = q.h1;
      l3.b[s] = weights->w3[s] + (size_t)m * q.h3 * q.h2;
      l3.n[s] = q.h3, l3.k[s] = q.h2, l3.ldb[s] = q.h2;
      l3t.b[s] = l3.b[s];                    // W3^T: B[n][k] = W3[k][n]
      l3t.n[s] = q.h2, l3t.k[s] = q.h3, l3t.ldb[s] = q.h2;
      l2t.b[s] = l2.b[s];                    // W2^T
      l2t.n[s] = q.h1, l2t.k[s] = q.h2, l2t.ldb[s] = q.h1;
    }
    const int32_t *ts = chunk->tile_species, *rs = chunk->row_slot;
    k_hessian_tangent_gemm<false, EPI_TANGENT><<<grid_g, 256, 0, st>>>(l1, jac, ldx, ts, rs, vec, hmax, VEC_S1, 0,
                                                                       nullptr, zd1, u, hmax);
    ANI_CUDA_CHECK_LAUNCH();
    k_hessian_tangent_gemm<false, EPI_TANGENT><<<grid_g, 256, 0, st>>>(l2, u, hmax, ts, rs, vec, hmax, VEC_S2, 0,
                                                                       nullptr, zd2, v, hmax);
    ANI_CUDA_CHECK_LAUNCH();
    k_hessian_tangent_gemm<false, EPI_SCALE><<<grid_g, 256, 0, st>>>(l3, v, hmax, ts, rs, vec, hmax, VEC_Q3, 0,
                                                                      nullptr, u, nullptr, hmax);
    ANI_CUDA_CHECK_LAUNCH();
    k_hessian_tangent_gemm<true, EPI_DELTA><<<grid_g, 256, 0, st>>>(l3t, u, hmax, ts, rs, vec, hmax, VEC_S2, VEC_R2,
                                                                     zd2, v, nullptr, hmax);
    ANI_CUDA_CHECK_LAUNCH();
    k_hessian_tangent_gemm<true, EPI_DELTA><<<grid_g, 256, 0, st>>>(l2t, v, hmax, ts, rs, vec, hmax, VEC_S1, VEC_R1,
                                                                     zd1, u, nullptr, hmax);
    ANI_CUDA_CHECK_LAUNCH();
    k_hessian_block_contract<<<dim3(chunk->n_slots, tiles * tiles), 256, 0, st>>>(
        zd1, u, hmax, nbr_cnt, cap, chunk->atom, chunk->row_off, chunk->block_off, sp4, *model, scale, blocks);
    ANI_CUDA_CHECK_LAUNCH();
  }
  return ANI_OK;
}

extern "C" int ani_b200_hessian_geometric(const ani_aev_params* params, const float* spos, const int32_t* nbr_cnt,
                                          const int32_t* nbr_list, int cap, const int32_t* row_of, const float* dx,
                                          int ldx, const ani_pair_params* pair_dev, const ani_hessian_chunk* chunk,
                                          float* blocks, void* stream) {
  if (!params || !spos || !nbr_cnt || !nbr_list || !blocks || cap < 1 || cap > 256) return ANI_ERR_BAD_ARG;
  if (!dx == !pair_dev || (dx && (!row_of || ldx % 32))) return ANI_ERR_BAD_ARG;
  if (int rc = check_chunk(chunk)) return rc;
  if (chunk->n_slots == 0) return ANI_OK;
  k_hessian_geometric<<<chunk->n_slots, 128, 0, (cudaStream_t)stream>>>(
      *params, reinterpret_cast<const float4*>(spos), nbr_cnt, nbr_list, cap, row_of, dx, ldx, pair_dev, chunk->atom,
      chunk->block_off, blocks);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_hessian_assemble(const int32_t* nbr_cnt, const int32_t* nbr_list, int cap,
                                         const int32_t* sorted_orig, const ani_hessian_chunk* chunk,
                                         const float* blocks, int n_per_conf, double* hess, void* stream) {
  if (!nbr_cnt || !nbr_list || !sorted_orig || !blocks || !hess || cap < 1 || cap > 256 || n_per_conf < 1)
    return ANI_ERR_BAD_ARG;
  if (int rc = check_chunk(chunk)) return rc;
  if (chunk->n_slots == 0) return ANI_OK;
  k_hessian_assemble<<<chunk->n_slots, 256, 0, (cudaStream_t)stream>>>(nbr_cnt, nbr_list, cap, sorted_orig,
                                                                       chunk->atom, chunk->block_off, blocks,
                                                                       n_per_conf, hess);
  ANI_CUDA_CHECK_LAUNCH();
  return ANI_OK;
}

extern "C" int ani_b200_hessian_hidden_max(const ani_mlp_model* model) {
  if (!model) return ANI_ERR_BAD_ARG;
  return max(model->h1_max, max(model->h2_max, model->h3_max));
}
