// Shared device helpers for the CUDA-native ANI hot path (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ani_b200.h"

#define ANI_WARP 32
#define ANI_FULL_MASK 0xffffffffu
#define ANI_IMG_SHIFT 26                       // neighbour word: sorted index | image code << 26
#define ANI_IDX_MASK ((1u << ANI_IMG_SHIFT) - 1u)

namespace ani {

// thread-local record of the last CUDA error (returned through the C-ABI)
void set_cuda_error(cudaError_t e);
#define ANI_CUDA_CHECK_LAUNCH()                         \
  do {                                                  \
    cudaError_t e__ = cudaGetLastError();               \
    if (e__ != cudaSuccess) {                           \
      ani::set_cuda_error(e__);                         \
      return ANI_ERR_CUDA;                              \
    }                                                   \
  } while (0)

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(ANI_FULL_MASK, v, o);
  return v;
}

// exp(x) for x <= 0 through ex2.approx (relative error ~2^-22 plus |x| * 2^-24 from the scaling):
// used for the Gaussian factors of the AEV, whose relevant range is x in [-16, 0]
__device__ __forceinline__ float fast_exp(float x) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * 1.4426950408889634f));
  return e;
}

// single-instruction MUFU forms (1-2 ulp): the IEEE-exact library versions cost 8-35 instructions
// each and sat on the issue-bound inner loops of the AEV kernels
__device__ __forceinline__ float fast_exp2(float x) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x));
  return e;
}
__device__ __forceinline__ float fast_log2(float x) {
  float e;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x));
  return e;
}
__device__ __forceinline__ float fast_rcp(float x) {
  float e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x));
  return e;
}
__device__ __forceinline__ float fast_sqrt(float x) {
  float e;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x));
  return e;
}

// index of the unordered species pair (a, b) in the row-major upper triangle of an SxS
// matrix (aev/_computer.py:184-191 == csrc/aev.cu:23-29)
__device__ __forceinline__ int pair_index(int a, int b, int S) {
  int lo = min(a, b), hi = max(a, b);
  return lo * (2 * S - lo + 1) / 2 + (hi - lo);
}

// cutoff function and derivative (cutoffs.py:70-101; derivative forms as aev.cu:141-178)
__device__ __forceinline__ float cutoff_value(float r, float rc, int kind) {
  if (kind == 0) return 0.5f * __cosf(r * (3.14159265358979323846f / rc)) + 0.5f;  // argument in [0, pi]: |err| < 5e-7
  float x = r / rc;
  float den = fmaxf(1e-10f, 1.0f - x * x);
  return expf(1.0f - 1.0f / den);
}

__device__ __forceinline__ void cutoff_value_grad(float r, float rc, int kind, float& f, float& df) {
  if (kind == 0) {
    float s, c;
    float a = 3.14159265358979323846f / rc;
    __sincosf(r * a, &s, &c);  // argument in [0, pi]
    f = 0.5f * c + 0.5f;
    df = -0.5f * a * s;
  } else {
    float x = r / rc;
    float one_m = 1.0f - x * x;
    if (one_m > 1e-10f) {
      f = expf(1.0f - 1.0f / one_m);
      df = f * (-2.0f * x / (rc * one_m * one_m));
    } else {
      f = expf(1.0f - 1e10f);
      df = 0.0f;
    }
  }
}

// image code (0..26) -> lattice shift vector.  code = (wx+1)*9 + (wy+1)*3 + (wz+1)
__device__ __forceinline__ float3 image_shift(const ani_grid& g, int code) {
  float wx = (float)(code / 9 - 1), wy = (float)((code / 3) % 3 - 1), wz = (float)(code % 3 - 1);
  float3 s;
  s.x = wx * g.cell[0] + wy * g.cell[3] + wz * g.cell[6];
  s.y = wx * g.cell[1] + wy * g.cell[4] + wz * g.cell[7];
  s.z = wx * g.cell[2] + wy * g.cell[5] + wz * g.cell[8];
  return s;
}

// grid mode 3 (one cell per conformer): the same shift in the lattice of conformer `conf`, from its row of the
// lattice table (ANI_LATTICE_STRIDE floats: cell, inverse)
__device__ __forceinline__ float3 image_shift(const float* __restrict__ lattice, int conf, int code) {
  const float* c = lattice + (size_t)conf * ANI_LATTICE_STRIDE;
  float wx = (float)(code / 9 - 1), wy = (float)((code / 3) % 3 - 1), wz = (float)(code % 3 - 1);
  float3 s;
  s.x = wx * c[0] + wy * c[3] + wz * c[6];
  s.y = wx * c[1] + wy * c[4] + wz * c[7];
  s.z = wx * c[2] + wy * c[5] + wz * c[8];
  return s;
}

// bucket b of a mode 0 / mode 2 / mode 3 grid -> its (ix, iy, iz) inside its sub-grid; returns the first bucket of that
// sub-grid (0 in mode 0; c * dims[0] * dims[1] * dims[2] for conformer c of a periodic batch)
__device__ __forceinline__ int bucket_coords(const ani_grid& g, int b, int& ix, int& iy, int& iz) {
  const int nb = g.dims[0] * g.dims[1] * g.dims[2];
  const int base = b - b % nb;
  b -= base;
  iz = b % g.dims[2];
  iy = (b / g.dims[2]) % g.dims[1];
  ix = b / (g.dims[2] * g.dims[1]);
  return base;
}

// ---- "tiled operand" layout shared by the AEV kernel (producer) and the tensor-core GEMM ----
// A matrix [rows][cols] is stored per 128-row tile and 32-column K-block as OPND_PARTS 16-bit
// pieces: [p1 128 rows x 64 B | p2 128 x 64 B (| p3)], every 8-row group in SWIZZLE_64B order
// (16-byte chunk c of row r sits at position c ^ ((r >> 1) & 3)).
//   ANI_OPND_FP16X2 = 1 (default): two IEEE half pieces of s*x (s = a power of two per operand
//     class, below), s*x = p1 + p2 with |residual| < 2^-22 |s*x| (two 11-bit significands):
//     4 B/element, three MMAs per product.  The scale keeps p2 out of the half subnormals for
//     every value that matters (absolute error < 2^-25 / s) and is divided out, exactly, in the
//     epilogue of the consuming GEMM.
//   ANI_OPND_FP16X2 = 0: three bfloat16 pieces x = p1 + p2 + p3 (no scale needed, 8-bit exponent):
//     6 B/element, six MMAs per product.
#ifndef ANI_OPND_FP16X2
#define ANI_OPND_FP16X2 1
#endif
constexpr int OPND_KB = 32;                                      // columns per K-block
constexpr int OPND_PARTS = ANI_OPND_FP16X2 ? 2 : 3;
constexpr int OPND_ROW_BYTES = 64;                               // 32 halves / bfloat16
constexpr int OPND_PART_BYTES = ANI_TILE_ROWS * OPND_ROW_BYTES;  // 8 KB
constexpr int OPND_BLOCK_BYTES = OPND_PARTS * OPND_PART_BYTES;   // 16 KB (24 KB for 3 x bf16)
// operand scales (powers of two).  Values: AEVs and CELU activations (|v| <= 65504 / 64 = 1023.5);
// gradients dE/d(activation) (|g| <= 65504 / 4096 = 15.9921875).  Weights carry a per-tensor scale
// chosen by the packer (ani_mlp_species::w_scale).  A producer that stores |s * v| > OPND_HALF_MAX
// (or a NaN, in the GEMM epilogues) raises ANI_STATUS_OPERAND_RANGE.
constexpr float OPND_SCALE_VALUE = ANI_OPND_FP16X2 ? 64.0f : 1.0f;
constexpr float OPND_SCALE_GRAD = ANI_OPND_FP16X2 ? 4096.0f : 1.0f;
constexpr float OPND_HALF_MAX = 65504.0f;
// byte offset of 16-byte chunk `ch` (0..3) of row `row` (0..127) inside one piece
__device__ __forceinline__ uint32_t swz_off(int row, int ch) {
  return (uint32_t)(row >> 3) * 512u + (uint32_t)(row & 7) * 64u + (uint32_t)((ch ^ ((row >> 1) & 3)) << 4);
}
// byte offset of element (row, col), piece 0, of a tiled matrix with `kblocks` = cols/32 blocks
// per row tile; piece k is k * OPND_PART_BYTES further
__device__ __forceinline__ size_t opnd_offset(int row, int col, int kblocks) {
  const int rt = row / ANI_TILE_ROWS, r = row % ANI_TILE_ROWS;
  return ((size_t)rt * kblocks + (col >> 5)) * OPND_BLOCK_BYTES + swz_off(r, (col & 31) >> 3) + (size_t)(col & 7) * 2;
}
// one value (already multiplied by its operand scale) -> OPND_PARTS 16-bit pieces (bit patterns)
__device__ __forceinline__ void opnd_split(float v, unsigned short (&p)[OPND_PARTS]) {
#if ANI_OPND_FP16X2
  auto rn = [](float x) -> unsigned short {
    unsigned short h;
    asm("cvt.rn.f16.f32 %0, %1;" : "=h"(h) : "f"(x));
    return h;
  };
  auto up = [](unsigned short h) -> float {
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(h));
    return f;
  };
  p[0] = rn(v);
  p[1] = rn(v - up(p[0]));
#else
  auto rn = [](float x) -> unsigned short {
    unsigned short h;
    asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(h) : "f"(x));
    return h;
  };
  p[0] = rn(v);
  v -= __uint_as_float((uint32_t)p[0] << 16);
  p[1] = rn(v);
  v -= __uint_as_float((uint32_t)p[1] << 16);
  p[2] = rn(v);
#endif
}

}  // namespace ani
