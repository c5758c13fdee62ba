// gemm_tc.cu — persistent wgmma implicit-GEMM convolution / linear kernel for sm_90a (H100).
//
//   384 threads = three warpgroups, warp-specialised. Warpgroup 0 is the producer: one thread feeds the STAGES-deep
//   shared-memory ring with TMA, cp.async.bulk.tensor 4-D (activations, shifted per tap, OOB zero fill = conv padding)
//   + 2-D (weights), and hands its registers to the consumers (setmaxnreg). Consumer warpgroup c = 1, 2 owns rows
//   [64(c-1), 64c) of the 128 x BN output tile and keeps its 64 x BN fp32 accumulator in registers (wgmma.m64nBNk16,
//   bf16 x bf16 -> fp32, both operands read from shared memory through SWIZZLE_128B descriptors), with one wgmma group
//   in flight while it waits for the next K block. The ring runs across tile boundaries, so the loads of a CTA's next
//   tile proceed while the consumers run the epilogue of the current one.
//   Epilogue: every warp moves its 16 rows through an XOR-swizzled 16 x 32 smem transpose, 32 columns at a time, to
//   fully coalesced global traffic (8 lanes own one 128-byte row segment) with fused bias / per-image vector / residual /
//   scale / accumulate / activation (SiLU, leaky-ReLU, GEGLU) / bf16 hi-lo split / GroupNorm statistics.
//
// See include/tango_b200.h (tng_conv_gemm) for the operator contract and the reference call sites it replaces.
#include "tng_ptx.cuh"
#include "tng_internal.h"
#include <stdlib.h>

namespace tng {

constexpr int BM = 128;
constexpr int BK = 64;  // bf16 elements per 128-byte swizzle row
constexpr int A_TILE_BYTES = BM * BK * 2;
constexpr int GEMM_THREADS = 384;
constexpr int EPI_WARPS = 8;
constexpr int ES = 4;   // epilogue row slots per lane: a warp's 16 rows = 4 slots x 4 row lanes

struct KGroupDev {
  int view, a_c0, dw, dh, b_k0, nkb;
};

struct GemmKernelParams {
  // output pixel grid and M tiling
  int W, H, NB;
  int bw, bh, bn;
  int tiles_w, tiles_h, tiles_n;
  int m_tiles, n_tiles;
  int Ncols;
  int n_groups, total_kiters;
  int ksplit;    // 1, or 2: two CTAs share an output tile, each reduces half of the K iterations and red.adds fp32 partials
  KGroupDev g[TNG_MAX_KGROUPS];
  // epilogue
  const float* bias;
  const float* rowvec;
  long long rowvec_ld;
  const void* res;
  int res_bf16;
  long long ldr;
  float alpha;
  int accumulate;
  float* out_f32;
  long long ld_f32;
  __nv_bfloat16* out_bf16;
  long long ld_bf16;
  int act;
  float act_param;
  int split_off;
  int vec_ok;    // all row strides / bases allow 16-byte vector access
  int fast_epi;  // vec_ok && Ncols % 4 == 0
  // GroupNorm statistics of the fp32 output, emitted from the epilogue (full-tile launches only, see the host side):
  // col_stats[(img * Ncols + col) * 2 + {0, 1}] += sum / sum of squares over the rows of image img = row / stats_hw
  double* col_stats;
  long long stats_hw;
};

template <int BN>
struct GemmCfg {
  static constexpr int B_TILE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_TILE_BYTES + B_TILE_BYTES;
  static constexpr int EPI_BYTES = EPI_WARPS * 16 * 32 * 4;  // per warp: 16 x 32 fp32 swizzled transpose tile
  static constexpr int STAGES_RAW = (227 * 1024 - EPI_BYTES - 256) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 256 /*barriers*/;
};

struct EpiRows {
  long long row[ES];
  int img[ES];
  uint32_t valid;
};

// One 16-row x 32-column chunk, already staged (swizzled) in `st`: lanes (rsub = lane >> 3, cg = lane & 7) own the
// 4 columns [4cg, 4cg+4) of rows 4i + rsub, i = 0..3.
template <bool RES, bool F32, bool BF16, bool VEC>
__device__ __forceinline__ void epi_chunk(const GemmKernelParams& p, const float* st, const EpiRows& R, int rsub, int cg,
                                          int col) {
  const bool col_ok = col < p.Ncols;
  const bool has_res = RES && (p.res != nullptr);
  const bool has_acc = F32 && (p.accumulate != 0);
  const bool has_f32 = F32 && (p.out_f32 != nullptr);
  const bool has_bf = BF16 && (p.out_bf16 != nullptr);
  // ---- all global loads of the chunk first (independent -> in flight together)
  float4 rres[ES], rold[ES];
  if (has_res) {
#pragma unroll
    for (int i = 0; i < ES; ++i) {
      float4 r4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (col_ok && ((R.valid >> i) & 1)) {
        if (VEC) {
          if (p.res_bf16) r4 = load_bf16x4(reinterpret_cast<const __nv_bfloat16*>(p.res) + R.row[i] * p.ldr + col);
          else r4 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.res) + R.row[i] * p.ldr + col);
        } else {
          float t[4] = {0.f, 0.f, 0.f, 0.f};
          for (int j = 0; j < 4; ++j)
            if (col + j < p.Ncols)
              t[j] = p.res_bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.res)[R.row[i] * p.ldr + col + j])
                                : reinterpret_cast<const float*>(p.res)[R.row[i] * p.ldr + col + j];
          r4 = make_float4(t[0], t[1], t[2], t[3]);
        }
      }
      rres[i] = r4;
    }
  }
  if (has_acc) {
#pragma unroll
    for (int i = 0; i < ES; ++i) {
      float4 r4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (col_ok && ((R.valid >> i) & 1)) {
        if (VEC) {
          r4 = *reinterpret_cast<const float4*>(p.out_f32 + R.row[i] * p.ld_f32 + col);
        } else {
          float t[4] = {0.f, 0.f, 0.f, 0.f};
          for (int j = 0; j < 4; ++j)
            if (col + j < p.Ncols) t[j] = p.out_f32[R.row[i] * p.ld_f32 + col + j];
          r4 = make_float4(t[0], t[1], t[2], t[3]);
        }
      }
      rold[i] = r4;
    }
  }
  float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (p.bias && col_ok) {
    if (VEC) {
      b4 = __ldg(reinterpret_cast<const float4*>(p.bias + col));
    } else {
      float t[4] = {0.f, 0.f, 0.f, 0.f};
      for (int j = 0; j < 4; ++j)
        if (col + j < p.Ncols) t[j] = __ldg(p.bias + col + j);
      b4 = make_float4(t[0], t[1], t[2], t[3]);
    }
  }
  const bool has_rv = (p.rowvec != nullptr);
  const float alpha = p.alpha;
#pragma unroll
  for (int i = 0; i < ES; ++i) {
    const int r = 4 * i + rsub;
    float4 a = *reinterpret_cast<const float4*>(st + r * 32 + ((cg ^ (r & 7)) << 2));
    if (!col_ok || !((R.valid >> i) & 1)) continue;
    a.x += b4.x; a.y += b4.y; a.z += b4.z; a.w += b4.w;
    if (has_rv) {
      const float* rv = p.rowvec + static_cast<long long>(R.img[i]) * p.rowvec_ld + col;
      if (VEC) {
        const float4 r4 = __ldg(reinterpret_cast<const float4*>(rv));
        a.x += r4.x; a.y += r4.y; a.z += r4.z; a.w += r4.w;
      } else {
        if (col + 0 < p.Ncols) a.x += __ldg(rv + 0);
        if (col + 1 < p.Ncols) a.y += __ldg(rv + 1);
        if (col + 2 < p.Ncols) a.z += __ldg(rv + 2);
        if (col + 3 < p.Ncols) a.w += __ldg(rv + 3);
      }
    }
    if (has_res) { a.x += rres[i].x; a.y += rres[i].y; a.z += rres[i].z; a.w += rres[i].w; }
    a.x *= alpha; a.y *= alpha; a.z *= alpha; a.w *= alpha;
    if (has_f32) {
      if (has_acc) { a.x += rold[i].x; a.y += rold[i].y; a.z += rold[i].z; a.w += rold[i].w; }
      float* op = p.out_f32 + R.row[i] * p.ld_f32 + col;
      if (VEC) {
        *reinterpret_cast<float4*>(op) = a;
      } else {
        const float t[4] = {a.x, a.y, a.z, a.w};
        for (int j = 0; j < 4; ++j)
          if (col + j < p.Ncols) op[j] = t[j];
      }
    }
    if (has_bf) {
      __nv_bfloat16* op = p.out_bf16 + R.row[i] * p.ld_bf16 + col;
      const float y0 = act_f(a.x, p.act, p.act_param), y1 = act_f(a.y, p.act, p.act_param);
      const float y2 = act_f(a.z, p.act, p.act_param), y3 = act_f(a.w, p.act, p.act_param);
      if (VEC) {
        store4_split(op, make_float4(y0, y1, y2, y3), p.split_off);
      } else {
        const float t[4] = {y0, y1, y2, y3};
        for (int j = 0; j < 4; ++j)
          if (col + j < p.Ncols) store_bf16_split(op + j, t[j], p.split_off);
      }
    }
  }
}

// Lean path for FULL tiles (all 128 rows valid, all 32 columns of the chunk < Ncols, 16-byte aligned): the rows of a
// tile are consecutive output rows (the host tiling guarantees it), so slot i of a lane is row r0 + 4i and every
// pointer advances by a constant stride — a few instructions per 16-byte access, no per-element predicates.
template <bool RES, bool F32, bool BF16>
__device__ __forceinline__ void epi_chunk_full(const GemmKernelParams& p, const float* st, long long r0, int img0,
                                               int rsub, int cg, int col, bool rv_uniform, long long stats_img) {
  float4 add4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (p.bias) add4 = __ldg(reinterpret_cast<const float4*>(p.bias + col));
  if (p.rowvec && rv_uniform) {
    const float4 r4 = __ldg(reinterpret_cast<const float4*>(p.rowvec + static_cast<long long>(img0) * p.rowvec_ld + col));
    add4.x += r4.x; add4.y += r4.y; add4.z += r4.z; add4.w += r4.w;
  }
  float4 rres[ES];
  if (RES) {
    if (p.res_bf16) {
      const __nv_bfloat16* rp = reinterpret_cast<const __nv_bfloat16*>(p.res) + r0 * p.ldr + col;
      const long long rs = 4 * p.ldr;
#pragma unroll
      for (int i = 0; i < ES; ++i) rres[i] = load_bf16x4(rp + i * rs);
    } else {
      const float* rp = reinterpret_cast<const float*>(p.res) + r0 * p.ldr + col;
      const long long rs = 4 * p.ldr;
#pragma unroll
      for (int i = 0; i < ES; ++i) rres[i] = *reinterpret_cast<const float4*>(rp + i * rs);
    }
  }
  float4 a[ES];
#pragma unroll
  for (int i = 0; i < ES; ++i) {
    const int r = 4 * i + rsub;
    a[i] = *reinterpret_cast<const float4*>(st + r * 32 + ((cg ^ (r & 7)) << 2));
    a[i].x += add4.x; a[i].y += add4.y; a[i].z += add4.z; a[i].w += add4.w;
  }
  if (p.rowvec && !rv_uniform) {
#pragma unroll
    for (int i = 0; i < ES; ++i) {
      const int im = img0 + (4 * i) / (p.bw * p.bh);  // img0 is the image of slot 0; rows advance by 4 per slot
      const float4 r4 = __ldg(reinterpret_cast<const float4*>(p.rowvec + static_cast<long long>(im) * p.rowvec_ld + col));
      a[i].x += r4.x; a[i].y += r4.y; a[i].z += r4.z; a[i].w += r4.w;
    }
  }
  if (RES) {
#pragma unroll
    for (int i = 0; i < ES; ++i) { a[i].x += rres[i].x; a[i].y += rres[i].y; a[i].z += rres[i].z; a[i].w += rres[i].w; }
  }
  if (p.alpha != 1.0f) {
    const float al = p.alpha;
#pragma unroll
    for (int i = 0; i < ES; ++i) { a[i].x *= al; a[i].y *= al; a[i].z *= al; a[i].w *= al; }
  }
  if (F32) {
    float* op = p.out_f32 + r0 * p.ld_f32 + col;
    const long long os = 4 * p.ld_f32;
    if (p.accumulate) {
#pragma unroll
      for (int i = 0; i < ES; ++i) {
        const float4 o4 = *reinterpret_cast<const float4*>(op + i * os);
        a[i].x += o4.x; a[i].y += o4.y; a[i].z += o4.z; a[i].w += o4.w;
      }
    }
#pragma unroll
    for (int i = 0; i < ES; ++i) *reinterpret_cast<float4*>(op + i * os) = a[i];
  }
  if (p.col_stats) {
    // Column sums of this warp's 16 rows x 32 columns (all rows belong to image stats_img): 4 rows in registers,
    // then across the four row-lanes (lane bits 3 and 4); lanes 0..7 hold the totals of their 4 columns and add
    // them to the fp64 per-(image, channel) accumulators — fp32 partials over 16 values, fp64 across tiles.
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f, q0 = 0.f, q1 = 0.f, q2 = 0.f, q3 = 0.f;
#pragma unroll
    for (int i = 0; i < ES; ++i) {
      s0 += a[i].x; s1 += a[i].y; s2 += a[i].z; s3 += a[i].w;
      q0 = fmaf(a[i].x, a[i].x, q0); q1 = fmaf(a[i].y, a[i].y, q1);
      q2 = fmaf(a[i].z, a[i].z, q2); q3 = fmaf(a[i].w, a[i].w, q3);
    }
#pragma unroll
    for (int o = 8; o <= 16; o <<= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o); s3 += __shfl_xor_sync(0xffffffffu, s3, o);
      q0 += __shfl_xor_sync(0xffffffffu, q0, o); q1 += __shfl_xor_sync(0xffffffffu, q1, o);
      q2 += __shfl_xor_sync(0xffffffffu, q2, o); q3 += __shfl_xor_sync(0xffffffffu, q3, o);
    }
    if (rsub == 0) {
      double* sp = p.col_stats + (stats_img * p.Ncols + col) * 2;
      atomicAdd(sp + 0, static_cast<double>(s0)); atomicAdd(sp + 1, static_cast<double>(q0));
      atomicAdd(sp + 2, static_cast<double>(s1)); atomicAdd(sp + 3, static_cast<double>(q1));
      atomicAdd(sp + 4, static_cast<double>(s2)); atomicAdd(sp + 5, static_cast<double>(q2));
      atomicAdd(sp + 6, static_cast<double>(s3)); atomicAdd(sp + 7, static_cast<double>(q3));
    }
  }
  if (BF16) {
    if (p.act == TNG_ACT_SILU) {
#pragma unroll
      for (int i = 0; i < ES; ++i) { a[i].x = silu_f(a[i].x); a[i].y = silu_f(a[i].y); a[i].z = silu_f(a[i].z); a[i].w = silu_f(a[i].w); }
    } else if (p.act == TNG_ACT_LRELU) {
      const float sl = p.act_param;
#pragma unroll
      for (int i = 0; i < ES; ++i) {
        a[i].x = a[i].x > 0.f ? a[i].x : a[i].x * sl; a[i].y = a[i].y > 0.f ? a[i].y : a[i].y * sl;
        a[i].z = a[i].z > 0.f ? a[i].z : a[i].z * sl; a[i].w = a[i].w > 0.f ? a[i].w : a[i].w * sl;
      }
    }
    __nv_bfloat16* op = p.out_bf16 + r0 * p.ld_bf16 + col;
    const long long os = 4 * p.ld_bf16;
#pragma unroll
    for (int i = 0; i < ES; ++i) store4_bf16(op + i * os, a[i]);
    if (p.split_off > 0) {
      op += p.split_off;
#pragma unroll
      for (int i = 0; i < ES; ++i) store4_bf16_lo(op + i * os, a[i]);
    }
  }
}

// 32 accumulator columns of this warp (8-column groups 4c .. 4c+3 = registers v[0, 16), see tng_ptx.cuh) -> the warp's
// 16 x 32 staging tile: row r at st + 32 r, its 16-byte unit u stored at unit u ^ (r & 7) (conflict-free reads above).
__device__ __forceinline__ void epi_stage(float* st, int lane, const float* v) {
  const int r = lane >> 2, t = lane & 3;
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int col = 8 * jj + 2 * t;
    const int off = (((col >> 2) ^ (r & 7)) << 2) + (col & 3);   // rows r and r + 8 share the swizzle phase
    *reinterpret_cast<float2*>(st + r * 32 + off) = make_float2(v[4 * jj], v[4 * jj + 1]);
    *reinterpret_cast<float2*>(st + (r + 8) * 32 + off) = make_float2(v[4 * jj + 2], v[4 * jj + 3]);
  }
}

// Stage chunk c (columns [32c, 32c + 32) of the tile) of the register accumulator. The accumulator is indexed with
// compile-time constants only (it must stay in registers), hence the unrolled select over the chunks.
template <int BN>
__device__ __forceinline__ void stage_chunk(float* st, int lane, const float (&acc)[BN / 2], int c) {
  __syncwarp();  // the previous chunk's smem reads are complete
#pragma unroll
  for (int cc = 0; cc < BN / 32; ++cc)
    if (cc == c) epi_stage(st, lane, acc + 16 * cc);
  __syncwarp();
}

template <int BN, bool RES, bool F32, bool BF16>
__device__ __forceinline__ void epi_tile_full(const GemmKernelParams& p, float* st, const float (&acc)[BN / 2], long long r0,
                                              int img0, bool rv_uniform, int tn, int lane, long long stats_img) {
  const int cg = lane & 7, rsub = lane >> 3;
#pragma unroll 1
  for (int c = 0; c < BN / 32; ++c) {
    stage_chunk<BN>(st, lane, acc, c);
    epi_chunk_full<RES, F32, BF16>(p, st, r0, img0, rsub, cg, tn * BN + 32 * c + 4 * cg, rv_uniform, stats_img);
  }
}

template <int BN, bool VEC>
__device__ __forceinline__ void epi_tile_generic(const GemmKernelParams& p, float* st, const float (&acc)[BN / 2],
                                                 const EpiRows& R, int tn, int lane) {
  const int cg = lane & 7, rsub = lane >> 3;
#pragma unroll 1
  for (int c = 0; c < BN / 32; ++c) {
    stage_chunk<BN>(st, lane, acc, c);
    epi_chunk<true, true, true, VEC>(p, st, R, rsub, cg, tn * BN + 32 * c + 4 * cg);
  }
}

// Split-K epilogue: this CTA holds the partial sum over its half of K. out (+)= alpha * (partial [+ bias + rowvec + res
// for the first half only]) with fp32 red.adds into an output the host zeroed beforehand. With exactly two partials
// per element the result does not depend on their order (0 + a + b, fp32 addition commutes), so runs stay
// reproducible. Used for under-filled launches with a long reduction (the 32x2 level of the UNet): the epilogue is
// small next to the main loop, so this is the simple row-slot form. wr = first tile row of this warp.
template <int BN>
__device__ __forceinline__ void epi_tile_splitk(const GemmKernelParams& p, float* st, const float (&acc)[BN / 2],
                                                long long row_base, int n0, int rpi, int nvalid, int sp, int tn, int lane,
                                                int wr) {
  const int cg = lane & 7, rsub = lane >> 3;
#pragma unroll 1
  for (int c = 0; c < BN / 32; ++c) {
    stage_chunk<BN>(st, lane, acc, c);
    const int col = tn * BN + 32 * c + 4 * cg;
    const bool col_ok = col < p.Ncols;   // Ncols % 4 == 0 (checked on the host)
    float4 add4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (col_ok && sp == 0 && p.bias) add4 = __ldg(reinterpret_cast<const float4*>(p.bias + col));
#pragma unroll 1
    for (int i = 0; i < ES; ++i) {
      const int rr = wr + 4 * i + rsub;
      if (!col_ok || rr >= nvalid) continue;
      const long long row = row_base + rr;
      float4 a = *reinterpret_cast<const float4*>(st + (4 * i + rsub) * 32 + ((cg ^ ((4 * i + rsub) & 7)) << 2));
      if (sp == 0) {
        a.x += add4.x; a.y += add4.y; a.z += add4.z; a.w += add4.w;
        if (p.rowvec) {
          const float4 r4 = __ldg(reinterpret_cast<const float4*>(p.rowvec + static_cast<long long>(n0 + rr / rpi) * p.rowvec_ld + col));
          a.x += r4.x; a.y += r4.y; a.z += r4.z; a.w += r4.w;
        }
        if (p.res) {
          if (p.res_bf16) {
            const float4 r4 = load_bf16x4(reinterpret_cast<const __nv_bfloat16*>(p.res) + row * p.ldr + col);
            a.x += r4.x; a.y += r4.y; a.z += r4.z; a.w += r4.w;
          } else {
            const float4 r4 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.res) + row * p.ldr + col);
            a.x += r4.x; a.y += r4.y; a.z += r4.z; a.w += r4.w;
          }
        }
      }
      a.x *= p.alpha; a.y *= p.alpha; a.z *= p.alpha; a.w *= p.alpha;
      float* op = p.out_f32 + row * p.ld_f32 + col;
      atomicAdd(op, a.x); atomicAdd(op + 1, a.y); atomicAdd(op + 2, a.z); atomicAdd(op + 3, a.w);
    }
  }
}

// GEGLU: columns [0, BN/2) of the tile are "hidden", [BN/2, BN) the matching "gate" (weights interleaved on the
// host). out[:, tn*BN/2 + j] = (hid + b) * gelu_erf(gate + b'). Rows r0 + 4i (consecutive-row tiles); rows >= nvalid
// are skipped.
template <int BN, bool FULL, bool SPLIT, bool TANH>
__device__ __forceinline__ void epi_tile_geglu(const GemmKernelParams& p, float* st, const float (&acc)[BN / 2], long long r0,
                                               int nleft, int tn, int lane) {
  constexpr int HALF = BN / 2;
  const int cg = lane & 7, rsub = lane >> 3;
#pragma unroll 1
  for (int c = 0; c < HALF / 32; ++c) {
    float4 hid[ES], g[ES];
    stage_chunk<BN>(st, lane, acc, c);
#pragma unroll
    for (int i = 0; i < ES; ++i) {
      const int r = 4 * i + rsub;
      hid[i] = *reinterpret_cast<const float4*>(st + r * 32 + ((cg ^ (r & 7)) << 2));
    }
    stage_chunk<BN>(st, lane, acc, c + HALF / 32);
#pragma unroll
    for (int i = 0; i < ES; ++i) {
      const int r = 4 * i + rsub;
      g[i] = *reinterpret_cast<const float4*>(st + r * 32 + ((cg ^ (r & 7)) << 2));
    }
    const int gcol = tn * BN + 32 * c + 4 * cg;  // GEMM column of the hidden half; gate at + HALF
    const int ocol = tn * HALF + 32 * c + 4 * cg;
    float4 bh = make_float4(0.f, 0.f, 0.f, 0.f), bg = bh;
    if (p.bias) {
      bh = __ldg(reinterpret_cast<const float4*>(p.bias + gcol));
      bg = __ldg(reinterpret_cast<const float4*>(p.bias + gcol + HALF));
    }
    // branch-free arithmetic over all 16 values of this lane (independent MUFU chains to interleave)
#pragma unroll
    for (int i = 0; i < ES; ++i) {
      hid[i].x = (hid[i].x + bh.x) * (TANH ? gelu_tanh_f(g[i].x + bg.x) : gelu_erf_f(g[i].x + bg.x));
      hid[i].y = (hid[i].y + bh.y) * (TANH ? gelu_tanh_f(g[i].y + bg.y) : gelu_erf_f(g[i].y + bg.y));
      hid[i].z = (hid[i].z + bh.z) * (TANH ? gelu_tanh_f(g[i].z + bg.z) : gelu_erf_f(g[i].z + bg.z));
      hid[i].w = (hid[i].w + bh.w) * (TANH ? gelu_tanh_f(g[i].w + bg.w) : gelu_erf_f(g[i].w + bg.w));
    }
    __nv_bfloat16* op = p.out_bf16 + r0 * p.ld_bf16 + ocol;
    const long long os = 4 * p.ld_bf16;
#pragma unroll
    for (int i = 0; i < ES; ++i) {
      if (!FULL && 4 * i >= nleft) continue;
      uint2 u;
      u.x = pack_bf16(hid[i].x, hid[i].y); u.y = pack_bf16(hid[i].z, hid[i].w);
      *reinterpret_cast<uint2*>(op + i * os) = u;
      if (SPLIT) {
        uint2 l;
        l.x = pack_bf16_lo(hid[i].x, hid[i].y); l.y = pack_bf16_lo(hid[i].z, hid[i].w);
        *reinterpret_cast<uint2*>(op + p.split_off + i * os) = l;
      }
    }
  }
}

// K iterations of work item `tile` (all of them unless split-K)
__device__ __forceinline__ int tile_kiters(const GemmKernelParams& p, int tile) {
  const int sp = tile % p.ksplit;
  return (sp + 1) * p.total_kiters / p.ksplit - sp * p.total_kiters / p.ksplit;
}

template <int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap amap0, const __grid_constant__ CUtensorMap amap1,
               const __grid_constant__ CUtensorMap amap2, const __grid_constant__ CUtensorMap amap3,
               const __grid_constant__ CUtensorMap bmap, const __grid_constant__ GemmKernelParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ __align__(1024) uint8_t smem[];  // SWIZZLE_128B tiles need 1024-byte alignment (checked below)
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_TILE_BYTES;
  float* sEpi = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES + Cfg::EPI_BYTES);  // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                                             // [STAGES]

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int wg = warp >> 2;

  if (tid == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();   // SWIZZLE_128B tiles need a 1024-byte aligned base
    tma_prefetch_desc(&amap0);
    tma_prefetch_desc(&bmap);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup once its wgmma reading the slot have completed
    }
    fence_mbar_init();
  }
  __syncthreads();

  // work items = (M tile, N tile[, K half]); split-K: consecutive work items are the K halves of one tile
  const int total_tiles = p.m_tiles * p.n_tiles * p.ksplit;
  const int work0 = blockIdx.x, work_stride = gridDim.x;

  if (wg == 0) {
    // ===================================================== TMA producer: the ring items of this CTA are its work items'
    // K blocks in order; item j lives in slot j % STAGES
    setmaxnreg_dec<40>();
    if (tid == 0) {
      uint32_t n_loaded = 0;
      for (int tile = work0; tile < total_tiles; tile += work_stride) {
        const int sp = tile % p.ksplit, t2 = tile / p.ksplit;
        const int tm = t2 / p.n_tiles, tn = t2 % p.n_tiles;
        const int tw = tm % p.tiles_w;
        const int th = (tm / p.tiles_w) % p.tiles_h;
        const int tb = tm / (p.tiles_w * p.tiles_h);
        const int w0 = tw * p.bw, h0 = th * p.bh, n0 = tb * p.bn;
        const int nk = tile_kiters(p, tile);
        int k = sp * p.total_kiters / p.ksplit, gi = 0;   // flat K iteration -> (k-group, K block)
        while (k >= p.g[gi].nkb) { k -= p.g[gi].nkb; ++gi; }
        for (int ki = 0; ki < nk; ++ki, ++k, ++n_loaded) {
          if (k == p.g[gi].nkb) { k = 0; ++gi; }
          const int slot = static_cast<int>(n_loaded % STAGES);
          const uint32_t use = n_loaded / STAGES;
          if (use > 0) mbar_wait(&empty_bar[slot], (use - 1) & 1);
          const KGroupDev g = p.g[gi];
          const CUtensorMap* am = g.view == 0 ? &amap0 : g.view == 1 ? &amap1 : g.view == 2 ? &amap2 : &amap3;
          mbar_arrive_expect_tx(&full_bar[slot], Cfg::STAGE_BYTES);
          tma_load_4d(sA + slot * A_TILE_BYTES, am, &full_bar[slot], g.a_c0 + k * BK, w0 + g.dw, h0 + g.dh, n0);
          tma_load_2d(sB + slot * Cfg::B_TILE_BYTES, &bmap, &full_bar[slot], g.b_k0 + k * BK, tn * BN);
        }
      }
    }
    return;
  }
  setmaxnreg_inc<232>();

  // ===================================================== main loop + epilogue (consumer warpgroups 1 and 2)
  const int cw = warp - 4;                         // consumer warp 0..7
  float* st = sEpi + cw * (16 * 32);
  const int rsub = lane >> 3;
  const int wr = 16 * cw;                          // first tile row of this warp
  const uint32_t a_off = static_cast<uint32_t>(wg - 1) * (64 * 128);   // rows [64 (wg-1), 64 wg) of the A tile
  const bool release = (tid & 127) == 0;           // the thread that arrives on the empty barriers for its warpgroup
  const int mode = (p.res ? 1 : 0) | (p.out_f32 ? 2 : 0) | (p.out_bf16 ? 4 : 0);
  const bool geglu = (p.act == TNG_ACT_GEGLU || p.act == TNG_ACT_GEGLU_TANH);
  uint32_t n_used = 0;                             // ring items consumed so far
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int tile = work0; tile < total_tiles; tile += work_stride) {
    const int sp = tile % p.ksplit, t2 = tile / p.ksplit;
    const int tm = t2 / p.n_tiles, tn = t2 % p.n_tiles;
    const int nk = tile_kiters(p, tile);
    for (int ki = 0; ki < nk; ++ki) {
      const int slot = static_cast<int>(n_used % STAGES);
      mbar_wait(&full_bar[slot], (n_used / STAGES) & 1);
      const uint64_t ad = wgmma_desc_sw128(smem_u32(sA + slot * A_TILE_BYTES) + a_off, 16, 1024);
      const uint64_t bd = wgmma_desc_sw128(smem_u32(sB + slot * Cfg::B_TILE_BYTES), 16, 1024);
      fence_regs(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) wgmma_ss<BN>(acc, ad + 2 * k, bd + 2 * k, (ki > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      fence_regs(acc);
      if (ki > 0) {
        wgmma_wait<1>();   // the previous K block's wgmma are complete: release its slot
        fence_regs(acc);
        mbar_arrive_if(&empty_bar[(n_used - 1) % STAGES], release);
      }
      ++n_used;
    }
    wgmma_wait<0>();
    fence_regs(acc);
    mbar_arrive_if(&empty_bar[(n_used - 1) % STAGES], release);

    // ---- epilogue: rows of a tile are consecutive output rows; valid rows form a prefix (see host tiling)
    const int tw = tm % p.tiles_w;
    const int th = (tm / p.tiles_w) % p.tiles_h;
    const int tb = tm / (p.tiles_w * p.tiles_h);
    const int w0 = tw * p.bw, h0 = th * p.bh, n0 = tb * p.bn;
    const long long row_base = (static_cast<long long>(n0) * p.H + h0) * p.W + w0;
    int nvalid;
    if (p.bh == 1 && p.bn == 1) nvalid = min(BM, p.W - w0);
    else if (p.bn == 1) nvalid = min(p.bh, p.H - h0) * p.bw;
    else nvalid = min(p.bn, p.NB - n0) * p.bh * p.bw;
    const int rpi = p.bw * p.bh;  // rows of one image inside a tile
    const bool full = p.fast_epi && (nvalid == BM) && ((tn + 1) * BN <= p.Ncols);
    if (p.ksplit > 1) {
      epi_tile_splitk<BN>(p, st, acc, row_base, n0, rpi, nvalid, sp, tn, lane, wr);
    } else if (geglu) {
      // slot i of this lane is row wr + rsub + 4i; rows below nvalid are valid
      if constexpr (BN == 128 || BN == 256) {   // the host only selects these N tiles for GEGLU
        const long long gr0 = row_base + wr + rsub;
        const int nleft = nvalid - (wr + rsub);
        if (p.act == TNG_ACT_GEGLU_TANH) {   // T5 front-end (small): one general instantiation
          if (p.split_off > 0) epi_tile_geglu<BN, false, true, true>(p, st, acc, gr0, nleft, tn, lane);
          else epi_tile_geglu<BN, false, false, true>(p, st, acc, gr0, nleft, tn, lane);
        } else if (p.split_off > 0) epi_tile_geglu<BN, false, true, false>(p, st, acc, gr0, nleft, tn, lane);
        else if (nvalid == BM) epi_tile_geglu<BN, true, false, false>(p, st, acc, gr0, nleft, tn, lane);
        else epi_tile_geglu<BN, false, false, false>(p, st, acc, gr0, nleft, tn, lane);
      }
    } else if (!full) {
      EpiRows R;
      R.valid = 0;
#pragma unroll
      for (int i = 0; i < ES; ++i) {
        const int rr = wr + 4 * i + rsub;
        R.img[i] = n0 + rr / rpi;
        R.row[i] = row_base + rr;
        if (rr < nvalid) R.valid |= 1u << i;
      }
      if (p.fast_epi) epi_tile_generic<BN, true>(p, st, acc, R, tn, lane);
      else epi_tile_generic<BN, false>(p, st, acc, R, tn, lane);
    } else {
      const long long r0 = row_base + wr + rsub;
      const int img0 = n0 + (wr + rsub) / rpi;
      const bool rv_uniform = (rpi % 16) == 0;   // the warp's 16 rows lie in one image
      // image of this warp's 16 consecutive output rows for the GroupNorm statistics (stats_hw % 16 == 0: host check)
      const long long simg = p.col_stats ? (row_base + wr) / p.stats_hw : 0;
      switch (mode) {
        case 2: epi_tile_full<BN, false, true, false>(p, st, acc, r0, img0, rv_uniform, tn, lane, simg); break;
        case 3: epi_tile_full<BN, true, true, false>(p, st, acc, r0, img0, rv_uniform, tn, lane, simg); break;
        case 4: epi_tile_full<BN, false, false, true>(p, st, acc, r0, img0, rv_uniform, tn, lane, simg); break;
        case 5: epi_tile_full<BN, true, false, true>(p, st, acc, r0, img0, rv_uniform, tn, lane, simg); break;
        case 6: epi_tile_full<BN, false, true, true>(p, st, acc, r0, img0, rv_uniform, tn, lane, simg); break;
        default: epi_tile_full<BN, true, true, true>(p, st, acc, r0, img0, rv_uniform, tn, lane, simg); break;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
template <int BN>
static int launch_gemm(const CUtensorMap* am, const CUtensorMap& bm, const GemmKernelParams& p, cudaStream_t st) {
  using Cfg = GemmCfg<BN>;
  const int rc = set_max_dynamic_smem<gemm_tc_kernel<BN>>(Cfg::SMEM_BYTES, "gemm_tc");
  if (rc) return rc;
  const int work = p.m_tiles * p.n_tiles * p.ksplit;
  const int grid = work < num_sms() ? work : num_sms();
  gemm_tc_kernel<BN><<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, st>>>(am[0], am[1], am[2], am[3], bm, p);
  return check_launch("gemm_tc");
}

static bool is_pow2(long long x) { return x > 0 && (x & (x - 1)) == 0; }

}  // namespace tng

using namespace tng;

// Everything that is decided before a launch: argument checks, the M tiling, the N tile, split-K and whether the
// GroupNorm statistics ride in the epilogue. Shared by tng_conv_gemm and tng_gemm_plan.
static int plan_gemm(const tng_gemm_desc* d, GemmKernelParams& p, int& bn_tile_out, bool& stats_after_out) {
  if (!d) return set_error(TNG_EINVAL, "null desc");
  if (d->n_aviews < 1 || d->n_aviews > TNG_MAX_AVIEWS) return set_error(TNG_EINVAL, "n_aviews=%d", d->n_aviews);
  if (d->n_groups < 1 || d->n_groups > TNG_MAX_KGROUPS) return set_error(TNG_EINVAL, "n_groups=%d", d->n_groups);
  if (d->W <= 0 || d->H <= 0 || d->NB <= 0 || d->Ncols <= 0) return set_error(TNG_EINVAL, "bad output grid");
  if ((d->ldb > 0 ? d->ldb : d->Ktot) % 8 != 0)
    return set_error(TNG_EINVAL, "B row stride must be a multiple of 8 elements (Ktot=%lld ldb=%lld)", (long long)d->Ktot, (long long)d->ldb);

  memset(&p, 0, sizeof(p));
  p.W = d->W; p.H = d->H; p.NB = d->NB;
  // M tile = bw x bh x bn output pixels (product 128)
  if (d->W >= BM || d->H == 1) {
    p.bw = BM; p.bh = 1; p.bn = 1;
  } else {
    if (!is_pow2(d->W)) return set_error(TNG_EINVAL, "W=%d < 128 must be a power of two", d->W);
    p.bw = d->W;
    const int rem = BM / p.bw;
    if (d->H >= rem) {
      p.bh = rem; p.bn = 1;
    } else {
      if (!is_pow2(d->H)) return set_error(TNG_EINVAL, "H=%d (W=%d) must be a power of two when W*H < 128", d->H, d->W);
      p.bh = d->H; p.bn = rem / p.bh;
    }
  }
  p.tiles_w = (d->W + p.bw - 1) / p.bw;
  p.tiles_h = (d->H + p.bh - 1) / p.bh;
  p.tiles_n = (d->NB + p.bn - 1) / p.bn;
  p.m_tiles = p.tiles_w * p.tiles_h * p.tiles_n;
  p.Ncols = (int)d->Ncols;

  int bn_tile = d->block_n;
  int ksplit = 1;
  if (d->act == TNG_ACT_GEGLU || d->act == TNG_ACT_GEGLU_TANH) {
    if (bn_tile == 0) bn_tile = (d->Ncols % 256 == 0) ? 256 : 128;
    if ((bn_tile != 128 && bn_tile != 256) || d->Ncols % bn_tile != 0 || !d->out_bf16 || d->out_f32 || d->res ||
        d->rowvec)
      return set_error(TNG_EINVAL, "GEGLU epilogue needs block_n 128/256 dividing Ncols, bf16 output only");
  }
  if (bn_tile == 0) {
    const long long N = d->Ncols;
    if (N <= 32) bn_tile = 32;
    else if (N <= 64) bn_tile = 64;
    else if (N % 256 == 0 && (long long)p.m_tiles * (N / 256) >= 2 * num_sms()) bn_tile = 256;
    else if (N % 160 == 0) {
      bn_tile = 160;
      // under-filled launches (e.g. the 32x2 level of the UNet: 8 M tiles)
      if ((long long)p.m_tiles * (N / 160) * 2 <= num_sms()) {
        static int splitk = -1;   // TNG_GEMM_SPLITK=0 disables (A/B measurements)
        if (splitk < 0) { const char* e = getenv("TNG_GEMM_SPLITK"); splitk = e ? atoi(e) : 1; }
        long long kit = 0;
        for (int i = 0; i < d->n_groups; ++i) kit += d->g[i].nkb;
        const bool can_split = splitk && d->out_f32 && !d->out_bf16 && !d->accumulate && d->act == TNG_ACT_NONE &&
                               d->res != d->out_f32 && kit >= 32 && d->Ncols % 4 == 0;
        if (can_split) ksplit = 2;   // two CTAs per output tile, each reduces half of K (long reductions only)
        else if (N % 128 == 0 && (long long)p.m_tiles * (N / 128) <= num_sms()) bn_tile = 128;  // more, smaller N tiles
      }
    }
    else if (N % 128 == 0) bn_tile = 128;
    else if (N % 64 == 0 && N < 256) bn_tile = 64;
    else bn_tile = 128;
  }
  p.n_tiles = (int)((d->Ncols + bn_tile - 1) / bn_tile);
  p.ksplit = ksplit;

  p.n_groups = d->n_groups;
  p.total_kiters = 0;
  for (int i = 0; i < d->n_groups; ++i) {
    const tng_kgroup& g = d->g[i];
    if (g.view < 0 || g.view >= d->n_aviews || g.nkb <= 0) return set_error(TNG_EINVAL, "k-group %d invalid", i);
    // The last K block may run past Ktot / the view's channel count: TMA zero-fills the out-of-range part of A,
    // so the (possibly non-zero) B columns read there contribute nothing.
    if (g.b_k0 < 0 || g.b_k0 + (long long)(g.nkb - 1) * BK >= d->Ktot)
      return set_error(TNG_EINVAL, "k-group %d: K block outside B", i);
    if (g.a_c0 < 0 || g.a_c0 + (long long)(g.nkb - 1) * BK >= d->a[g.view].C)
      return set_error(TNG_EINVAL, "k-group %d: K block outside view channels", i);
    p.g[i] = KGroupDev{g.view, g.a_c0, g.dw, g.dh, g.b_k0, g.nkb};
    p.total_kiters += g.nkb;
  }
  p.bias = d->bias; p.rowvec = d->rowvec; p.rowvec_ld = d->rowvec_ld > 0 ? d->rowvec_ld : d->Ncols; p.res = d->res; p.res_bf16 = (d->res_dtype == TNG_DT_BF16);
  p.ldr = d->ldr; p.alpha = d->alpha; p.accumulate = d->accumulate;
  p.out_f32 = d->out_f32; p.ld_f32 = d->ld_f32;
  p.out_bf16 = reinterpret_cast<__nv_bfloat16*>(d->out_bf16); p.ld_bf16 = d->ld_bf16;
  p.act = d->act; p.act_param = d->act_param; p.split_off = d->split_off;
  if (!d->out_f32 && !d->out_bf16) return set_error(TNG_EINVAL, "no output");
  if (d->accumulate && !d->out_f32) return set_error(TNG_EINVAL, "accumulate needs out_f32");

  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  bool vec = true;
  if (d->bias && !al16(d->bias)) vec = false;
  if (d->rowvec && (!al16(d->rowvec) || p.rowvec_ld % 4)) vec = false;
  if (d->res) {
    if (!al16(d->res)) vec = false;
    if (p.res_bf16 ? (d->ldr % 8) : (d->ldr % 4)) vec = false;
  }
  if (d->out_f32 && (!al16(d->out_f32) || d->ld_f32 % 4)) vec = false;
  if (d->out_bf16 && (!al16(d->out_bf16) || d->ld_bf16 % 8 || d->split_off % 8)) vec = false;
  p.vec_ok = vec ? 1 : 0;
  p.fast_epi = (vec && d->Ncols % 4 == 0) ? 1 : 0;
  if ((d->act == TNG_ACT_GEGLU || d->act == TNG_ACT_GEGLU_TANH) && !vec) return set_error(TNG_EINVAL, "GEGLU epilogue needs 16-byte aligned output");
  if (d->gn_stats) {
    if (d->stats_hw <= 0 || (static_cast<long long>(d->W) * d->H * d->NB) % d->stats_hw != 0)
      return set_error(TNG_EINVAL, "gn_stats: the output rows must be whole images of stats_hw pixels");
    if (!d->out_f32 && (d->split_off > 0 || d->act != TNG_ACT_NONE))
      return set_error(TNG_EINVAL, "gn_stats without an fp32 output needs a plain bf16 output (no activation, no hi/lo split)");
  }

  const bool full_m = (p.bh == 1 && p.bn == 1) ? (d->W % BM == 0) : (p.bn == 1 ? (d->H % p.bh == 0) : (d->NB % p.bn == 0));
  if (p.ksplit > 1 && !p.fast_epi) p.ksplit = 1;
  // GroupNorm statistics ride in the epilogue when every tile is full (the lean epilogue path), the warp's 16 rows lie
  // in one image and the output is written exactly once; otherwise a separate pass over the output follows the GEMM
  bool stats_after = false;
  if (d->gn_stats) {
    const bool fused = full_m && (d->Ncols % bn_tile == 0) && p.fast_epi && p.ksplit == 1 && !d->accumulate &&
                       (d->stats_hw % 16 == 0) && d->act != TNG_ACT_GEGLU && d->act != TNG_ACT_GEGLU_TANH;
    if (fused) { p.col_stats = d->gn_stats; p.stats_hw = d->stats_hw; }
    else stats_after = true;
  }
  bn_tile_out = bn_tile;
  stats_after_out = stats_after;
  return TNG_OK;
}

extern "C" int tng_gemm_plan(const tng_gemm_desc* d, int32_t* block_n, int32_t* mode, int32_t* ksplit) {
  GemmKernelParams p;
  int bn_tile = 0;
  bool stats_after = false;
  const int rc = plan_gemm(d, p, bn_tile, stats_after);
  if (rc != TNG_OK) return rc;
  if (block_n) *block_n = bn_tile;
  if (mode) *mode = 1;
  if (ksplit) *ksplit = p.ksplit;
  return TNG_OK;
}

extern "C" int tng_conv_gemm(const tng_gemm_desc* d, void* stream) {
  GemmKernelParams p;
  int bn_tile = 0;
  bool stats_after = false;
  {
    const int rc = plan_gemm(d, p, bn_tile, stats_after);
    if (rc != TNG_OK) return rc;
  }
  // tensor maps
  CUtensorMap am[4];
  for (int i = 0; i < 4; ++i) {
    const tng_aview& v = d->a[i < d->n_aviews ? i : 0];
    if (v.C % 8 != 0) return set_error(TNG_EINVAL, "view %d: C=%lld must be a multiple of 8", i, (long long)v.C);
    uint64_t dims[4] = {(uint64_t)v.C, (uint64_t)v.W, (uint64_t)v.H, (uint64_t)v.NB};
    uint64_t strides[3] = {(uint64_t)v.s_w * 2, (uint64_t)v.s_h * 2, (uint64_t)v.s_n * 2};
    uint32_t box[4] = {(uint32_t)BK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
    int rc = encode_tmap_bf16(&am[i], v.ptr, 4, dims, strides, box);
    if (rc) return rc;
  }
  CUtensorMap bm;
  {
    uint64_t dims[2] = {(uint64_t)d->Ktot, (uint64_t)d->Ncols};
    uint64_t strides[1] = {(uint64_t)(d->ldb > 0 ? d->ldb : d->Ktot) * 2};
    uint32_t box[2] = {(uint32_t)BK, (uint32_t)bn_tile};
    int rc = encode_tmap_bf16(&bm, d->b, 2, dims, strides, box);
    if (rc) return rc;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (p.ksplit > 1) {   // the partial sums are red.added into a zeroed output
    const size_t rows = static_cast<size_t>(d->W) * d->H * d->NB;
    cudaError_t e = cudaMemset2DAsync(d->out_f32, static_cast<size_t>(d->ld_f32) * 4, 0, static_cast<size_t>(d->Ncols) * 4, rows, st);
    if (e != cudaSuccess) return set_error(TNG_ECUDA, "cudaMemset2DAsync(split-K output): %s", cudaGetErrorString(e));
  }
  int rc;
  switch (bn_tile) {
    case 32: rc = launch_gemm<32>(am, bm, p, st); break;
    case 64: rc = launch_gemm<64>(am, bm, p, st); break;
    case 128: rc = launch_gemm<128>(am, bm, p, st); break;
    case 160: rc = launch_gemm<160>(am, bm, p, st); break;
    case 256: rc = launch_gemm<256>(am, bm, p, st); break;
    default: return set_error(TNG_EINVAL, "block_n=%d unsupported", bn_tile);
  }
  if (rc == TNG_OK && stats_after) {
    const long long rows = static_cast<long long>(d->W) * d->H * d->NB;
    // (from the stored output: fp32 when there is one, else the bf16 output — the rounded values the consumer reads)
    if (d->out_f32) rc = launch_col_stats(d->out_f32, TNG_DT_F32, d->Ncols, d->ld_f32, rows / d->stats_hw, d->stats_hw, d->gn_stats, st);
    else rc = launch_col_stats(d->out_bf16, TNG_DT_BF16, d->Ncols, d->ld_bf16, rows / d->stats_hw, d->stats_hw, d->gn_stats, st);
  }
  return rc;
}
