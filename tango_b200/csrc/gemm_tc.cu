// gemm_tc.cu — persistent wgmma implicit-GEMM convolution / linear kernel for sm_90a (H100).
//
//   384 threads = three warpgroups, warp-specialised. Warpgroup 0 is the producer: one thread feeds the STAGES-deep
//   shared-memory ring with TMA, cp.async.bulk.tensor 4-D (activations, shifted per tap, OOB zero fill = conv padding)
//   + 2-D (weights), and hands its registers to the consumers (setmaxnreg). Consumer warpgroup c = 1, 2 owns rows
//   [BM/2 (c-1), BM/2 c) of the BM x BN output tile and keeps its BM/2 x BN fp32 accumulator in registers, one
//   wgmma.m64nBNk16 per 64 rows (bf16 x bf16 -> fp32, both operands read from shared memory through SWIZZLE_128B
//   descriptors; the 64-row halves of a 256-row tile share the B descriptor), with one wgmma group in flight while it
//   waits for the next K block. BM = 128, or 256 with BN = 160 (28 % fewer operand bytes per FLOP than 128 x 160; see
//   plan_gemm for when). The ring runs across tile boundaries, so the loads of a CTA's next tile proceed while the
//   consumers run the epilogue of the current one.
//   Epilogue: every warp moves its 16 rows through an XOR-swizzled 16 x 32 smem transpose, 32 columns at a time, to
//   fully coalesced global traffic (8 lanes own one 128-byte row segment) with fused bias / per-image vector / residual /
//   scale / accumulate / activation (SiLU, leaky-ReLU, GEGLU) / bf16 hi-lo split / GroupNorm statistics.
//
// See include/tango_b200.h (tng_conv_gemm) for the operator contract and the reference call sites it replaces.
#include "tng_ptx.cuh"
#include "tng_internal.h"

namespace tng {

constexpr int BK = 64;  // bf16 elements per 128-byte swizzle row
constexpr int GEMM_THREADS = 384;
constexpr int EPI_WARPS = 8;
constexpr int ES = 4;   // epilogue row slots per lane: a warp's 16 rows = 4 slots x 4 row lanes

struct KGroupDev {
  int view, a_c0, dw, dh, b_k0, nkb;
};

struct GemmKernelParams {
  // output pixel grid and M tiling
  int W, H, NB;
  int bw, bh, bn;   // M tile = bw x bh x bn output pixels, bm = their product (128 or 256)
  int bm;
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
  int fast_epi;  // Ncols % 4 == 0 and every epilogue row stride and base allows 16-byte vector access
  // GroupNorm statistics of the stored output, emitted from the epilogue (full-tile launches only, see the host side):
  // col_stats[(img * Ncols + col) * 2 + {0, 1}] += sum / sum of squares over the rows of image img = row / stats_hw
  double* col_stats;
  long long stats_hw;
};

template <int BN, int BM>
struct GemmCfg {
  static constexpr int A_TILE_BYTES = BM * BK * 2;
  static constexpr int B_TILE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_TILE_BYTES + B_TILE_BYTES;
  static constexpr int EPI_BYTES = EPI_WARPS * 16 * 32 * 4;  // per warp: 16 x 32 fp32 swizzled transpose tile
  static constexpr int STAGES_RAW = (227 * 1024 - EPI_BYTES - 256) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 256 /*barriers*/;
};

// Chunk shapes of the epilogue (epi_tile). FULL: every row slot and column of the chunk is valid and 16-byte aligned,
// fixed at compile time, so the code carries no predicates. VEC: 16-byte accesses, rows and columns predicated (partial
// tiles, split-K). SCALAR: one access per element (Ncols % 4 != 0 or misaligned operands).
enum EpiShape { EPI_SCALAR, EPI_VEC, EPI_FULL };

__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 scale4(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

// act_f over a chunk, with the activation fixed at compile time
template <int ACT>
__device__ __forceinline__ void act_chunk(float4 (&a)[ES], float ap) {
#pragma unroll
  for (int i = 0; i < ES; ++i)
    a[i] = make_float4(act_f(a[i].x, ACT, ap), act_f(a[i].y, ACT, ap), act_f(a[i].z, ACT, ap), act_f(a[i].w, ACT, ap));
}

// Row r, columns [4cg, 4cg + 4) of a warp's 16 x 32 staging tile (layout: epi_stage)
__device__ __forceinline__ float4 staged(const float* st, int r, int cg) {
  return *reinterpret_cast<const float4*>(st + r * 32 + ((cg ^ (r & 7)) << 2));
}

// The first n (<= 4) values at q (fp32 or bf16) as fp32, zero-filled; one vector load when VEC (n is 4 there). RO
// reads through the read-only cache: bias and rowvec only, never the residual or the old output, which the kernel may
// be writing.
template <bool VEC, bool RO = false, typename T>
__device__ __forceinline__ float4 load4(const T* q, int n) {
  if constexpr (VEC && sizeof(T) == 2) return load_bf16x4(q);
  if constexpr (VEC && sizeof(T) == 4)
    return RO ? __ldg(reinterpret_cast<const float4*>(q)) : *reinterpret_cast<const float4*>(q);
  float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (j < n) t[j] = static_cast<float>(RO ? __ldg(q + j) : q[j]);
  return make_float4(t[0], t[1], t[2], t[3]);
}

template <bool VEC>
__device__ __forceinline__ float4 load_bias(const GemmKernelParams& p, int col, int n) {
  return p.bias ? load4<VEC, true>(p.bias + col, n) : make_float4(0.f, 0.f, 0.f, 0.f);
}

// the residual at element offset off
template <bool VEC>
__device__ __forceinline__ float4 load_res(const GemmKernelParams& p, long long off, int n) {
  return p.res_bf16 ? load4<VEC>(static_cast<const __nv_bfloat16*>(p.res) + off, n)
                    : load4<VEC>(static_cast<const float*>(p.res) + off, n);
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

// The current work item as the epilogue sees it: the tile's rows are the consecutive output rows starting at row_base,
// of which the first nvalid are valid (see the host tiling); tile row r lies in image n0 + r / (bw * bh). tn = N tile,
// sp = K half under split-K.
struct EpiTile {
  long long row_base;
  int n0, nvalid, tn, sp;
};

// Epilogue of one non-GEGLU tile, 32 columns per chunk. MODE bits: 1 residual, 2 fp32 output, 4 bf16 output. FULL tiles
// compile in exactly the parts the launch uses; the other shapes compile in all three and test the pointers.
// Lane (rsub = lane >> 3, cg = lane & 7) owns columns [col, col + 4) of tile rows wr + rsub + 4i, i < ES:
//   out = ((((acc + bias) + rowvec[image]) + res) * alpha) [+ out when accumulating]
// Split-K: each K half red.adds alpha * its partial into an fp32 output the host zeroed, and only half 0 adds the bias,
// rowvec and residual. With exactly two partials per element the result does not depend on their order (0 + a + b,
// fp32 addition commutes), so runs stay reproducible.
// All global loads of a chunk are issued before its first store: res may be out_f32 (the transformer out-projections).
template <int BN, int SHAPE, int MODE>
__device__ __forceinline__ void epi_tile(const GemmKernelParams& p, float* st, const float (&acc)[BN / 2], const EpiTile& t,
                                         int wr, int lane) {
  constexpr bool FULL = SHAPE == EPI_FULL, VEC = SHAPE != EPI_SCALAR;
  const int cg = lane & 7, rsub = lane >> 3;
  const int trow = wr + rsub;                 // tile row of slot 0
  const long long r0 = t.row_base + trow;     // output row of slot 0
  const int lane_rows = FULL ? ES : min(ES, max(0, (t.nvalid - trow + 3) >> 2));   // valid slots: a prefix
  const bool red = SHAPE == EPI_VEC && p.ksplit > 1;   // split-K tiles: never FULL, always 16-byte aligned (host)
  const bool add_terms = !red || t.sp == 0;
  const bool has_res = (MODE & 1) && (FULL || p.res) && add_terms;
  const bool has_f32 = (MODE & 2) && (FULL || p.out_f32);
  const bool has_bf = (MODE & 4) && (FULL || p.out_bf16);
  const bool has_rv = p.rowvec && add_terms;
  const int rpi = p.bw * p.bh;   // rows of one image inside a tile: a power of two (host tiling)
  const int rpi_log2 = __ffs(rpi) - 1;
  // image of the warp's 16 rows for the GroupNorm statistics (stats_hw % 16 == 0: host check)
  const long long simg = (FULL && p.col_stats) ? (t.row_base + wr) / p.stats_hw : 0;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
  for (int c = 0; c < BN / 32; ++c) {
    stage_chunk<BN>(st, lane, acc, c);
    const int col = t.tn * BN + 32 * c + 4 * cg;
    const int ncols = FULL ? 4 : min(4, p.Ncols - col);   // valid columns of the lane, none when <= 0
    const int nrows = ncols > 0 ? lane_rows : 0;
    float4 res[ES];
    if (has_res) {
      const long long off = r0 * p.ldr + col, rs = 4 * p.ldr;
#pragma unroll
      for (int i = 0; i < ES; ++i) res[i] = i < nrows ? load_res<VEC>(p, off + i * rs, ncols) : zero;
    }
    const float4 b4 = (add_terms && ncols > 0) ? load_bias<VEC>(p, col, ncols) : zero;
    // branch-free, so that the four staging reads issue together (one branch between them costs ~5 % on the
    // HBM-bound GEMMs)
    float4 a[ES];
#pragma unroll
    for (int i = 0; i < ES; ++i) a[i] = add4(staged(st, 4 * i + rsub, cg), b4);
    if (has_rv) {
      float4 rv = zero;
#pragma unroll
      for (int i = 0; i < ES; ++i) {
        if (i >= nrows) continue;
        // image n0 + (tile row) / rpi; when rpi % 16 == 0 the warp's 16 rows lie in one image, loaded by slot 0
        const long long img = t.n0 + ((trow + 4 * i) >> rpi_log2);
        if (i == 0 || rpi % 16 != 0) rv = load4<VEC, true>(p.rowvec + img * p.rowvec_ld + col, ncols);
        a[i] = add4(a[i], rv);
      }
    }
#pragma unroll
    for (int i = 0; i < ES; ++i) a[i] = scale4(has_res ? add4(a[i], res[i]) : a[i], p.alpha);
    if (has_f32) {
      float* op = p.out_f32 + r0 * p.ld_f32 + col;
      const long long os = 4 * p.ld_f32;
      if (p.accumulate) {
#pragma unroll
        for (int i = 0; i < ES; ++i)
          if (i < nrows) a[i] = add4(a[i], load4<VEC>(op + i * os, ncols));
      }
#pragma unroll
      for (int i = 0; i < ES; ++i) {
        if (i >= nrows) continue;
        float* q = op + i * os;
        if (red) {
          atomicAdd(q, a[i].x); atomicAdd(q + 1, a[i].y); atomicAdd(q + 2, a[i].z); atomicAdd(q + 3, a[i].w);
        } else if (VEC) {
          *reinterpret_cast<float4*>(q) = a[i];
        } else {
          const float v[4] = {a[i].x, a[i].y, a[i].z, a[i].w};
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (j < ncols) q[j] = v[j];
        }
      }
    }
    if (FULL && p.col_stats) {
      // Column sums of this warp's 16 rows x 32 columns (all rows belong to image simg): 4 rows in registers,
      // then across the four row-lanes (lane bits 3 and 4); lanes 0..7 hold the totals of their 4 columns and add
      // them to the fp64 per-(image, channel) accumulators — fp32 partials over 16 values, fp64 across tiles.
      // Without an fp32 output they are the statistics of the stored bf16 values (a plain bf16 output: host check),
      // as the after-pass computes them.
      float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f, q0 = 0.f, q1 = 0.f, q2 = 0.f, q3 = 0.f;
#pragma unroll
      for (int i = 0; i < ES; ++i) {
        float4 v = a[i];
        if constexpr (!(MODE & 2)) v = make_float4(bf16_round(v.x), bf16_round(v.y), bf16_round(v.z), bf16_round(v.w));
        s0 += v.x; s1 += v.y; s2 += v.z; s3 += v.w;
        q0 = fmaf(v.x, v.x, q0); q1 = fmaf(v.y, v.y, q1);
        q2 = fmaf(v.z, v.z, q2); q3 = fmaf(v.w, v.w, q3);
      }
#pragma unroll
      for (int o = 8; o <= 16; o <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o); s3 += __shfl_xor_sync(0xffffffffu, s3, o);
        q0 += __shfl_xor_sync(0xffffffffu, q0, o); q1 += __shfl_xor_sync(0xffffffffu, q1, o);
        q2 += __shfl_xor_sync(0xffffffffu, q2, o); q3 += __shfl_xor_sync(0xffffffffu, q3, o);
      }
      if (rsub == 0) {
        double* sp = p.col_stats + (simg * p.Ncols + col) * 2;
        atomicAdd(sp + 0, static_cast<double>(s0)); atomicAdd(sp + 1, static_cast<double>(q0));
        atomicAdd(sp + 2, static_cast<double>(s1)); atomicAdd(sp + 3, static_cast<double>(q1));
        atomicAdd(sp + 4, static_cast<double>(s2)); atomicAdd(sp + 5, static_cast<double>(q2));
        atomicAdd(sp + 6, static_cast<double>(s3)); atomicAdd(sp + 7, static_cast<double>(q3));
      }
    }
    if (has_bf) {
      // one branch on p.act per chunk: a branch per element makes the bf16-output GEMMs ~30 % slower
      if (p.act == TNG_ACT_SILU) act_chunk<TNG_ACT_SILU>(a, p.act_param);
      else if (p.act == TNG_ACT_LRELU) act_chunk<TNG_ACT_LRELU>(a, p.act_param);
      __nv_bfloat16* op = p.out_bf16 + r0 * p.ld_bf16 + col;
      const long long os = 4 * p.ld_bf16;
#pragma unroll
      for (int i = 0; i < ES; ++i) {
        if (i >= nrows) continue;
        if (VEC) {
          store4_bf16(op + i * os, a[i]);
        } else {
          const float v[4] = {a[i].x, a[i].y, a[i].z, a[i].w};
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (j < ncols) store_bf16_split(op + i * os + j, v[j], p.split_off);
        }
      }
      if (VEC && p.split_off > 0) {
#pragma unroll
        for (int i = 0; i < ES; ++i)
          if (i < nrows) store4_bf16_lo(op + p.split_off + i * os, a[i]);
      }
    }
  }
}

// GEGLU: columns [0, BN/2) of the tile are "hidden", [BN/2, BN) the matching "gate" (weights interleaved on the
// host). out[:, tn*BN/2 + j] = (hid + b) * gelu_erf(gate + b'). Rows past nvalid are skipped unless FULL.
template <int BN, bool FULL, bool SPLIT, bool TANH>
__device__ __forceinline__ void epi_tile_geglu(const GemmKernelParams& p, float* st, const float (&acc)[BN / 2],
                                               const EpiTile& t, int wr, int lane) {
  constexpr int HALF = BN / 2;
  const int cg = lane & 7, rsub = lane >> 3;
  const int trow = wr + rsub;
#pragma unroll 1
  for (int c = 0; c < HALF / 32; ++c) {
    float4 hid[ES], g[ES];
    stage_chunk<BN>(st, lane, acc, c);
#pragma unroll
    for (int i = 0; i < ES; ++i) hid[i] = staged(st, 4 * i + rsub, cg);
    stage_chunk<BN>(st, lane, acc, c + HALF / 32);
#pragma unroll
    for (int i = 0; i < ES; ++i) g[i] = staged(st, 4 * i + rsub, cg);
    const int gcol = t.tn * BN + 32 * c + 4 * cg;  // GEMM column of the hidden half; gate at + HALF
    const int ocol = t.tn * HALF + 32 * c + 4 * cg;
    const float4 bh = load_bias<true>(p, gcol, 4), bg = load_bias<true>(p, gcol + HALF, 4);
    // branch-free arithmetic over all 16 values of this lane (independent MUFU chains to interleave)
#pragma unroll
    for (int i = 0; i < ES; ++i) {
      hid[i].x = (hid[i].x + bh.x) * (TANH ? gelu_tanh_f(g[i].x + bg.x) : gelu_erf_f(g[i].x + bg.x));
      hid[i].y = (hid[i].y + bh.y) * (TANH ? gelu_tanh_f(g[i].y + bg.y) : gelu_erf_f(g[i].y + bg.y));
      hid[i].z = (hid[i].z + bh.z) * (TANH ? gelu_tanh_f(g[i].z + bg.z) : gelu_erf_f(g[i].z + bg.z));
      hid[i].w = (hid[i].w + bh.w) * (TANH ? gelu_tanh_f(g[i].w + bg.w) : gelu_erf_f(g[i].w + bg.w));
    }
    __nv_bfloat16* op = p.out_bf16 + (t.row_base + trow) * p.ld_bf16 + ocol;
    const long long os = 4 * p.ld_bf16;
#pragma unroll
    for (int i = 0; i < ES; ++i) {
      if (!FULL && trow + 4 * i >= t.nvalid) continue;
      store4_bf16(op + i * os, hid[i]);
      if (SPLIT) store4_bf16_lo(op + p.split_off + i * os, hid[i]);
    }
  }
}

// Work item `tile` (under split-K consecutive items are the K halves of one output tile): K half sp, N tile tn and the
// origin (w0, h0, n0) of its M tile in the output pixel grid
struct WorkItem {
  int sp, tn, w0, h0, n0;
};
__device__ __forceinline__ WorkItem work_item(const GemmKernelParams& p, int tile) {
  const int t2 = tile / p.ksplit, tm = t2 / p.n_tiles;
  const int tw = tm % p.tiles_w, th = (tm / p.tiles_w) % p.tiles_h, tb = tm / (p.tiles_w * p.tiles_h);
  return WorkItem{tile % p.ksplit, t2 % p.n_tiles, tw * p.bw, th * p.bh, tb * p.bn};
}

// K iterations of work item `tile` (all of them unless split-K)
__device__ __forceinline__ int tile_kiters(const GemmKernelParams& p, int tile) {
  const int sp = tile % p.ksplit;
  return (sp + 1) * p.total_kiters / p.ksplit - sp * p.total_kiters / p.ksplit;
}

template <int BN, int BM>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap amap0, const __grid_constant__ CUtensorMap amap1,
               const __grid_constant__ CUtensorMap amap2, const __grid_constant__ CUtensorMap amap3,
               const __grid_constant__ CUtensorMap bmap, const __grid_constant__ GemmKernelParams p) {
  using Cfg = GemmCfg<BN, BM>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int A_TILE_BYTES = Cfg::A_TILE_BYTES;
  constexpr int MH = BM / 128;   // 64-row accumulator blocks per consumer warpgroup
  // register split (128 x 24 + 256 x 240 <= 64K): 256-row tiles keep 160 accumulators per consumer thread, and the
  // producer's one thread fits in 24 registers
  constexpr int PRODUCER_REGS = BM == 256 ? 24 : 40, CONSUMER_REGS = BM == 256 ? 240 : 232;
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
    setmaxnreg_dec<PRODUCER_REGS>();
    if (tid == 0) {
      uint32_t n_loaded = 0;
      for (int tile = work0; tile < total_tiles; tile += work_stride) {
        const WorkItem w = work_item(p, tile);
        const int nk = tile_kiters(p, tile);
        int k = w.sp * p.total_kiters / p.ksplit, gi = 0;   // flat K iteration -> (k-group, K block)
        while (k >= p.g[gi].nkb) { k -= p.g[gi].nkb; ++gi; }
        for (int ki = 0; ki < nk; ++ki, ++k, ++n_loaded) {
          if (k == p.g[gi].nkb) { k = 0; ++gi; }
          const int slot = static_cast<int>(n_loaded % STAGES);
          const uint32_t use = n_loaded / STAGES;
          if (use > 0) mbar_wait(&empty_bar[slot], (use - 1) & 1);
          const KGroupDev g = p.g[gi];
          const CUtensorMap* am = g.view == 0 ? &amap0 : g.view == 1 ? &amap1 : g.view == 2 ? &amap2 : &amap3;
          mbar_arrive_expect_tx(&full_bar[slot], Cfg::STAGE_BYTES);
          tma_load_4d(sA + slot * A_TILE_BYTES, am, &full_bar[slot], g.a_c0 + k * BK, w.w0 + g.dw, w.h0 + g.dh, w.n0);
          tma_load_2d(sB + slot * Cfg::B_TILE_BYTES, &bmap, &full_bar[slot], g.b_k0 + k * BK, w.tn * BN);
        }
      }
    }
    return;
  }
  setmaxnreg_inc<CONSUMER_REGS>();

  // ===================================================== main loop + epilogue (consumer warpgroups 1 and 2)
  const int cw = warp - 4;                         // consumer warp 0..7
  float* st = sEpi + cw * (16 * 32);
  // first tile row of this warp in each 64-row block of its warpgroup: wr0 + 64 h, h < MH (the wgmma accumulator
  // layout gives warp i of a warpgroup rows [16 i, 16 i + 16) of every m64 block)
  const int wr0 = (BM / 2) * (wg - 1) + 16 * (cw & 3);
  const uint32_t a_off = static_cast<uint32_t>(wg - 1) * (BM / 2 * 128);   // rows [BM/2 (wg-1), BM/2 wg) of the A tile
  const bool release = (tid & 127) == 0;           // the thread that arrives on the empty barriers for its warpgroup
  uint32_t n_used = 0;                             // ring items consumed so far
  float acc[MH][BN / 2];
#pragma unroll
  for (int h = 0; h < MH; ++h)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
  for (int tile = work0; tile < total_tiles; tile += work_stride) {
    const int nk = tile_kiters(p, tile);
    for (int ki = 0; ki < nk; ++ki) {
      const int slot = static_cast<int>(n_used % STAGES);
      mbar_wait(&full_bar[slot], (n_used / STAGES) & 1);
      const uint32_t sa = smem_u32(sA + slot * A_TILE_BYTES) + a_off;
      const uint64_t bd = wgmma_desc_sw128(smem_u32(sB + slot * Cfg::B_TILE_BYTES), 16, 1024);
#pragma unroll
      for (int h = 0; h < MH; ++h) fence_regs(acc[h]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
#pragma unroll
        for (int h = 0; h < MH; ++h)
          wgmma_ss<BN>(acc[h], wgmma_desc_sw128(sa + h * (64 * 128), 16, 1024) + 2 * k, bd + 2 * k,
                       (ki > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
#pragma unroll
      for (int h = 0; h < MH; ++h) fence_regs(acc[h]);
      if (ki > 0) {
        wgmma_wait<1>();   // the previous K block's wgmma are complete: release its slot
#pragma unroll
        for (int h = 0; h < MH; ++h) fence_regs(acc[h]);
        mbar_arrive_if(&empty_bar[(n_used - 1) % STAGES], release);
      }
      ++n_used;
    }
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < MH; ++h) fence_regs(acc[h]);
    mbar_arrive_if(&empty_bar[(n_used - 1) % STAGES], release);

    // ---- epilogue: rows of a tile are consecutive output rows; valid rows form a prefix (see host tiling)
    const WorkItem w = work_item(p, tile);
    int nvalid;
    if (p.bh == 1 && p.bn == 1) nvalid = min(BM, p.W - w.w0);
    else if (p.bn == 1) nvalid = min(p.bh, p.H - w.h0) * p.bw;
    else nvalid = min(p.bn, p.NB - w.n0) * p.bh * p.bw;
    const EpiTile t{(static_cast<long long>(w.n0) * p.H + w.h0) * p.W + w.w0, w.n0, nvalid, w.tn, w.sp};
    const int mode = (p.res ? 1 : 0) | (p.out_f32 ? 2 : 0) | (p.out_bf16 ? 4 : 0);
    const bool geglu = (p.act == TNG_ACT_GEGLU || p.act == TNG_ACT_GEGLU_TANH);
    const bool full = p.fast_epi && p.ksplit == 1 && nvalid == BM && (w.tn + 1) * BN <= p.Ncols;
#pragma unroll
    for (int h = 0; h < MH; ++h) {
      const int wr = wr0 + 64 * h;
      if (geglu) {
        if constexpr (BM == 128 && (BN == 128 || BN == 256)) {   // the host only selects these tiles for GEGLU
          if (p.act == TNG_ACT_GEGLU_TANH) {   // T5 front-end (small): one general instantiation
            if (p.split_off > 0) epi_tile_geglu<BN, false, true, true>(p, st, acc[h], t, wr, lane);
            else epi_tile_geglu<BN, false, false, true>(p, st, acc[h], t, wr, lane);
          } else if (p.split_off > 0) epi_tile_geglu<BN, false, true, false>(p, st, acc[h], t, wr, lane);
          else if (nvalid == BM) epi_tile_geglu<BN, true, false, false>(p, st, acc[h], t, wr, lane);
          else epi_tile_geglu<BN, false, false, false>(p, st, acc[h], t, wr, lane);
        }
      } else if (full) {
        switch (mode) {
          case 2: epi_tile<BN, EPI_FULL, 2>(p, st, acc[h], t, wr, lane); break;
          case 3: epi_tile<BN, EPI_FULL, 3>(p, st, acc[h], t, wr, lane); break;
          case 4: epi_tile<BN, EPI_FULL, 4>(p, st, acc[h], t, wr, lane); break;
          case 5: epi_tile<BN, EPI_FULL, 5>(p, st, acc[h], t, wr, lane); break;
          case 6: epi_tile<BN, EPI_FULL, 6>(p, st, acc[h], t, wr, lane); break;
          default: epi_tile<BN, EPI_FULL, 7>(p, st, acc[h], t, wr, lane); break;
        }
      } else if (p.fast_epi) {
        epi_tile<BN, EPI_VEC, 7>(p, st, acc[h], t, wr, lane);
      } else if constexpr (BM == 128) {   // 256-row tiles: 16-byte aligned operands only (host)
        epi_tile<BN, EPI_SCALAR, 7>(p, st, acc[h], t, wr, lane);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
template <int BN, int BM = 128>
static int launch_gemm(const CUtensorMap* am, const CUtensorMap& bm, const GemmKernelParams& p, cudaStream_t st) {
  using Cfg = GemmCfg<BN, BM>;
  const int rc = set_max_dynamic_smem<gemm_tc_kernel<BN, BM>>(Cfg::SMEM_BYTES, "gemm_tc");
  if (rc) return rc;
  const int work = p.m_tiles * p.n_tiles * p.ksplit;
  const int grid = work < num_sms() ? work : num_sms();
  gemm_tc_kernel<BN, BM><<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, st>>>(am[0], am[1], am[2], am[3], bm, p);
  return check_launch("gemm_tc");
}

static bool is_pow2(long long x) { return x > 0 && (x & (x - 1)) == 0; }

// M tile = bw x bh x bn output pixels with product bm (a power of two), each box dimension <= bm <= 256 (the TMA box
// limit): whole rows of the output grid when W >= bm, else whole images' worth of rows, so that the rows of a tile are
// consecutive output rows and its valid rows a prefix. False when the grid does not allow this tiling.
static bool tile_m(const tng_gemm_desc* d, int bm, GemmKernelParams& p) {
  if (d->W >= bm || d->H == 1) {
    p.bw = bm; p.bh = 1; p.bn = 1;
  } else {
    if (!is_pow2(d->W)) return false;
    p.bw = d->W;
    const int rem = bm / p.bw;
    if (d->H >= rem) {
      p.bh = rem; p.bn = 1;
    } else {
      if (!is_pow2(d->H)) return false;
      p.bh = d->H; p.bn = rem / p.bh;
    }
  }
  p.tiles_w = (d->W + p.bw - 1) / p.bw;
  p.tiles_h = (d->H + p.bh - 1) / p.bh;
  p.tiles_n = (d->NB + p.bn - 1) / p.bn;
  p.m_tiles = p.tiles_w * p.tiles_h * p.tiles_n;
  p.bm = bm;
  return true;
}

// every M tile of the tiling in p is full
static bool full_m_tiles(const tng_gemm_desc* d, const GemmKernelParams& p) {
  return (p.bh == 1 && p.bn == 1) ? (d->W % p.bw == 0) : (p.bn == 1 ? (d->H % p.bh == 0) : (d->NB % p.bn == 0));
}

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
  if (!tile_m(d, 128, p)) {
    if (!is_pow2(d->W)) return set_error(TNG_EINVAL, "W=%d < 128 must be a power of two", d->W);
    return set_error(TNG_EINVAL, "H=%d (W=%d) must be a power of two when W*H < 128", d->H, d->W);
  }
  p.Ncols = (int)d->Ncols;

  int bn_tile = d->block_n;
  int ksplit = 1;
  if (d->act == TNG_ACT_GEGLU || d->act == TNG_ACT_GEGLU_TANH) {
    if (bn_tile == 0) bn_tile = (d->Ncols % 256 == 0) ? 256 : 128;
    if ((bn_tile != 128 && bn_tile != 256) || d->Ncols % bn_tile != 0 || !d->out_bf16 || d->out_f32 || d->res ||
        d->rowvec)
      return set_error(TNG_EINVAL, "GEGLU epilogue needs block_n 128/256 dividing Ncols, bf16 output only");
    // epi_tile_geglu applies the bias only: a scale would have to act on both halves before the GELU
    if (d->alpha != 1.0f) return set_error(TNG_EINVAL, "GEGLU epilogue needs alpha = 1 (alpha=%g)", (double)d->alpha);
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
        long long kit = 0;
        for (int i = 0; i < d->n_groups; ++i) kit += d->g[i].nkb;
        const bool can_split = d->out_f32 && !d->out_bf16 && !d->accumulate && d->act == TNG_ACT_NONE &&
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
  p.fast_epi = (vec && d->Ncols % 4 == 0) ? 1 : 0;
  if ((d->act == TNG_ACT_GEGLU || d->act == TNG_ACT_GEGLU_TANH) && !vec) return set_error(TNG_EINVAL, "GEGLU epilogue needs 16-byte aligned output");
  if (d->gn_stats) {
    if (d->stats_hw <= 0 || (static_cast<long long>(d->W) * d->H * d->NB) % d->stats_hw != 0)
      return set_error(TNG_EINVAL, "gn_stats: the output rows must be whole images of stats_hw pixels");
    if (!d->out_f32 && (d->split_off > 0 || d->act != TNG_ACT_NONE))
      return set_error(TNG_EINVAL, "gn_stats without an fp32 output needs a plain bf16 output (no activation, no hi/lo split)");
  }

  if (p.ksplit > 1 && !p.fast_epi) p.ksplit = 1;
  // 256-row tiles draw 28 % fewer operand bytes from L2 per FLOP than 128 x 160, but a CTA's epilogue covers twice the
  // rows and a launch has half the work items. On one H100 SXM (700 W) that pays for long reductions only: 3x3
  // convolutions with >= 1280 input channels gain up to 5 %; short-K linears (K = 320 / 640) with an fp32 residual lose
  // 6-12 % and the level-0 3x3 convolution (K = 2880) 3 % (DESIGN.md section 7). So: non-GEGLU (GEGLU's epilogue works
  // on 128 x 256 tiles), not split-K, 16-byte aligned epilogue operands, >= 64 K blocks, and at least half a wave of
  // 256-row work items; with fused statistics only when every 256-row tile is full.
  if (bn_tile == 160 && p.ksplit == 1 && p.fast_epi && p.total_kiters >= 64 && d->act != TNG_ACT_GEGLU &&
      d->act != TNG_ACT_GEGLU_TANH) {
    GemmKernelParams q = p;
    if (tile_m(d, 256, q) && 2LL * q.m_tiles * p.n_tiles >= num_sms() && (!d->gn_stats || full_m_tiles(d, q))) p = q;
  }
  const bool full_m = full_m_tiles(d, p);
  // GroupNorm statistics ride in the epilogue when every tile is full (the lean epilogue path), the warp's 16 rows lie
  // in one image and the output is written exactly once; otherwise a separate pass over the output follows the GEMM
  bool stats_after = false;
  if (d->gn_stats) {
    const bool fused = full_m && (d->Ncols % bn_tile == 0) && p.fast_epi && p.ksplit == 1 && !d->accumulate &&
                       (d->stats_hw % 16 == 0) && d->act != TNG_ACT_GEGLU && d->act != TNG_ACT_GEGLU_TANH;
    if (fused) { p.col_stats = d->gn_stats; p.stats_hw = d->stats_hw; }
    else stats_after = true;
    // the after-pass (launch_col_stats) reads the stored output 4 columns at a time: refuse before the GEMM runs what
    // it would refuse after the GEMM has written the output
    const void* so = d->out_f32 ? static_cast<const void*>(d->out_f32) : d->out_bf16;
    const long long sld = d->out_f32 ? d->ld_f32 : d->ld_bf16;
    if (stats_after && (d->Ncols % 4 || sld % 4 || (reinterpret_cast<uintptr_t>(so) & 7)))
      return set_error(TNG_EINVAL, "gn_stats after the GEMM needs Ncols %% 4 == 0 and a stored output with ld %% 4 == 0, "
                       "8-byte aligned (Ncols=%lld ld=%lld)", (long long)d->Ncols, sld);
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
  if (mode) *mode = p.bm;
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
    uint32_t box[4] = {(uint32_t)BK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};   // bm x BK
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
    case 160: rc = p.bm == 256 ? launch_gemm<160, 256>(am, bm, p, st) : launch_gemm<160>(am, bm, p, st); break;
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
