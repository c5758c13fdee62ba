// attention.cu — wgmma flash attention, sm_90a: the UNet's self- and cross-attention (head width 64) and the AudioLDM
// VAE AttnBlock (audioldm/variational_autoencoder/modules.py:204-230: ONE head of width 512 over the H*W positions of
// an image, 4096 positions for a 10 s clip, 12288 for 30 s). The score matrix never leaves the SM.
//
// One CTA = 128 query rows x DV value / output columns of one batch entry: consumer warpgroup g owns query rows
// [64g, 64g + 64). Q / K / V arrive as TMA SWIZZLE_128B chunks of 64 columns (Q once; K / V in tiles of 64 keys, NBUF
// buffers deep). With NBUF > 1 a ninth warp (288 threads) is the producer: one of its lanes issues every load and
// refills a K / V buffer as soon as both warpgroups have released it, so the consumers only wait for data and the
// warpgroups can drift up to NBUF - 1 tiles apart (one's softmax then runs while the other's wgmma keep the tensor
// cores busy).
// Per key tile: S = Q K^T over the D/64 head chunks (wgmma m64n64k16, both operands K-major in shared memory)
// -> fp32 online softmax in registers (the four lanes that share a row combine their maxima / sums by shuffles)
// -> O += P V with P taken straight from registers as the A operand (the accumulator layout of S is the A-fragment
// layout) and V consumed as an MN-major B operand (no transpose), 64 output columns per instruction.
//
//   <64, 64, 1, 3>    head width 64, bf16 operands: 64 KB of shared memory, two CTAs per SM. 18 warps put 5 on one
//                     SM sub-partition, whose 16 K registers leave 96 per thread; the consumers fit without spills.
//   <64, 64, 2, 3>    the parity mode: every operand carries its bf16 rounding residual and each product is evaluated as
//                     hi*hi + lo*hi + hi*lo, which restores ~fp32 accuracy on the bf16 tensor cores (1 CTA / SM).
//   <512, 256, 1, 1>  the VAE: Q [128 x 512] (128 KB) + K [64 x 512] (64 KB) + V [64 x 256] (32 KB) = 224 KB, which is
//                     why K / V are single-buffered and refilled in line by thread 0 (with a producer warp, 3 warps on
//                     one sub-partition would leave 168 registers per thread, and the kernel needs 197). O [64 x 256]
//                     takes 128 fp32 registers per thread, so a CTA computes one half of V / O and both halves
//                     recompute S (the score FLOPs double; they are 1/5 of a decoder that is itself < 1 % of a
//                     200-step generation). bf16 only: the VAE's parity mode keeps the
//                     GEMM -> softmax -> GEMM formulation.
// The key mask, the ragged last key tile, rows past Lq and the lo half of the output are features of the head-64 entry;
// the VAE entry has none of them (no mask, L a multiple of 128, bf16 output).
#include "tng_ptx.cuh"
#include "tng_internal.h"

namespace tng {

constexpr int FA_BM = 128;                // queries per CTA
constexpr int FA_BN = 64;                 // keys per tile
constexpr int FA_QCHUNK = FA_BM * 128;    // one [128][64] bf16 swizzled chunk = 16 KB
constexpr int FA_KCHUNK = FA_BN * 128;    // one [64][64] bf16 swizzled chunk = 8 KB
constexpr int FA_CONSUMERS = 256;        // two warpgroups
// + the producer warp when the K / V ring is more than one buffer deep
constexpr int fa_threads(int nbuf) { return nbuf > 1 ? FA_CONSUMERS + 32 : FA_CONSUMERS; }
// Exponentials of the head-64 bf16 entry that run on the FMA pipe (ex2_poly) instead of MUFU: every FA_POLY_EVERY-th
// of each row, 0 = none. A 64-key tile costs as many MUFU clocks (4096 ex2 at 16 / clk / SM) as tensor clocks, but the
// kernel is bound by instruction issue, not by MUFU: ex2_poly is 10 instructions where ex2.approx is one. At B = 16,
// 5 heads, 4096 x 4096 (H100 80GB HBM3, 700 W) every 4th exponential on ex2_poly made the kernel 894 us against 793 us
// with none; before the scale was folded into the exponent's FMA, every 4th / 3rd / 2nd took it from 957 us to 1068 /
// 1090 / 1178 us.
constexpr int FA_POLY_EVERY = 0;

struct AttnParams {
  int Lq, Lk;
  int q_col0, q_lo_off, k_col0, k_lo_off, v_col0, v_lo_off;
  const float* kbias;
  __nv_bfloat16* out;
  long long ld_o;
  int split_off;
  float scale_log2e;  // scale * log2(e)
};

template <int D, int DV, int NSPLIT, int NBUF>
struct FlashCfg {
  static constexpr int Q_BYTES = NSPLIT * (D / 64) * FA_QCHUNK;
  static constexpr int K_BYTES = NSPLIT * (D / 64) * FA_KCHUNK;    // per buffer
  static constexpr int V_BYTES = NSPLIT * (DV / 64) * FA_KCHUNK;   // per buffer
  static constexpr int SMEM_BYTES = Q_BYTES + NBUF * (K_BYTES + V_BYTES) + 128;
  static_assert((1 + 4 * NBUF) * 8 <= 128, "the mbarriers fit the 128 bytes after the tiles");
  static_assert(SMEM_BYTES <= 227 * 1024, "an H100 CTA has at most 227 KB of dynamic shared memory");
};

template <int D, int DV, int NSPLIT, int NBUF>
__global__ void __launch_bounds__(fa_threads(NBUF), (D == 64 && NSPLIT == 1) ? 2 : 1)
flash_attention_kernel(const __grid_constant__ CUtensorMap qmap, const __grid_constant__ CUtensorMap kmap,
                       const __grid_constant__ CUtensorMap vmap, const __grid_constant__ AttnParams p) {
  using Cfg = FlashCfg<D, DV, NSPLIT, NBUF>;
  constexpr int DC = D / 64, NV = DV / 64;   // 64-column chunks of a Q / K row and of a V / O row
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;                                // [NSPLIT][DC] chunks
  uint8_t* sK = sQ + Cfg::Q_BYTES;                   // [NBUF][NSPLIT][DC]
  uint8_t* sV = sK + NBUF * Cfg::K_BYTES;            // [NBUF][NSPLIT][NV]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + NBUF * Cfg::V_BYTES);
  uint64_t* bar_q = bars;                            // [1]
  uint64_t* full_k = bars + 1;                       // [NBUF] K tile landed
  uint64_t* full_v = bars + 1 + NBUF;                // [NBUF] V tile landed
  uint64_t* empty_k = bars + 1 + 2 * NBUF;           // [NBUF] both warpgroups are done with the K buffer
  uint64_t* empty_v = bars + 1 + 3 * NBUF;           // [NBUF] ... with the V buffer

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int wg = warp >> 2;
  const int q0 = blockIdx.x * FA_BM;
  const int b = blockIdx.z;
  const int n_tiles = (p.Lk + FA_BN - 1) / FA_BN;
  // blockIdx.y is a column slice: Q / K start y * D columns in when DV = D and at 0 otherwise, V / O start y * DV in.
  // For head width 64 it is the head; for the VAE it is the half of V / O this CTA computes over the whole head.
  const int qk_col = blockIdx.y * (DV == D ? D : 0);
  const int vo_col = blockIdx.y * DV;

  auto load_k = [&](int t) {
    const int buf = t % NBUF;
    mbar_arrive_expect_tx(&full_k[buf], Cfg::K_BYTES);
#pragma unroll
    for (int s = 0; s < NSPLIT; ++s)
#pragma unroll
      for (int c = 0; c < DC; ++c)
        tma_load_3d(sK + buf * Cfg::K_BYTES + (s * DC + c) * FA_KCHUNK, &kmap, &full_k[buf],
                    p.k_col0 + s * p.k_lo_off + qk_col + 64 * c, t * FA_BN, b);
  };
  auto load_v = [&](int t) {
    const int buf = t % NBUF;
    mbar_arrive_expect_tx(&full_v[buf], Cfg::V_BYTES);
#pragma unroll
    for (int s = 0; s < NSPLIT; ++s)
#pragma unroll
      for (int c = 0; c < NV; ++c)
        tma_load_3d(sV + buf * Cfg::V_BYTES + (s * NV + c) * FA_KCHUNK, &vmap, &full_v[buf],
                    p.v_col0 + s * p.v_lo_off + vo_col + 64 * c, t * FA_BN, b);
  };

  constexpr bool PRODUCER = NBUF > 1;
  if (tid == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();   // SWIZZLE_128B tiles need a 1024-byte aligned base
    tma_prefetch_desc(&qmap);
    tma_prefetch_desc(&kmap);
    tma_prefetch_desc(&vmap);
    mbar_init(bar_q, 1);
    for (int i = 0; i < NBUF; ++i) {
      mbar_init(&full_k[i], 1);
      mbar_init(&full_v[i], 1);
      mbar_init(&empty_k[i], 2);
      mbar_init(&empty_v[i], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();
  auto load_q = [&] {
    mbar_arrive_expect_tx(bar_q, Cfg::Q_BYTES);
#pragma unroll
    for (int s = 0; s < NSPLIT; ++s)
#pragma unroll
      for (int c = 0; c < DC; ++c)
        tma_load_3d(sQ + (s * DC + c) * FA_QCHUNK, &qmap, bar_q, p.q_col0 + s * p.q_lo_off + qk_col + 64 * c, q0, b);
  };
  if (!PRODUCER && tid == 0) {
    load_q();
    load_k(0);
    load_v(0);
  }

  if (PRODUCER && tid >= FA_CONSUMERS) {   // ---- the producer warp: Q once, then the K / V ring
    if (tid == FA_CONSUMERS) {
      load_q();
      for (int t = 0; t < n_tiles; ++t) {
        // buffer t % NBUF last held tile t - NBUF; both warpgroups release its K after S and its V after PV
        const uint32_t ph = ((t / NBUF) & 1) ^ 1;
        if (t >= NBUF) mbar_wait(&empty_k[t % NBUF], ph);
        load_k(t);
        if (t >= NBUF) mbar_wait(&empty_v[t % NBUF], ph);
        load_v(t);
      }
    }
    return;
  }

  constexpr int NT = (NSPLIT == 1) ? 1 : 3;   // split products: hi*hi, lo*hi, hi*lo
  const int qsel[3] = {0, 1, 0}, ksel[3] = {0, 0, 1};
  const uint32_t q_base = smem_u32(sQ) + wg * (64 * 128);   // this warpgroup's 64 query rows
  const uint32_t k_base = smem_u32(sK), v_base = smem_u32(sV);
  const float sc = p.scale_log2e;
  constexpr float LOG2E = 1.4426950408889634f;
  const float* kb = p.kbias ? p.kbias + static_cast<long long>(b) * p.Lk : nullptr;
  const int t4 = lane & 3;
  // this thread holds rows rA = (lane >> 2) and rA + 8 of its warp's 16 rows; columns 8j + 2 t4 + {0, 1}
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
  float o[NV][32];
#pragma unroll
  for (int n = 0; n < NV; ++n)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[n][i] = 0.f;

  mbar_wait(bar_q, 0);
  for (int t = 0; t < n_tiles; ++t) {
    const int buf = t % NBUF;
    const uint32_t ph = (t / NBUF) & 1;
    // ---- S = Q K^T over the 64 keys of tile t
    float s[32];
    mbar_wait(&full_k[buf], ph);
    fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int u = 0; u < NT; ++u) {
#pragma unroll
      for (int c = 0; c < DC; ++c) {
        const uint64_t qd = wgmma_desc_sw128(q_base + (qsel[u] * DC + c) * FA_QCHUNK, 16, 1024);
        const uint64_t kd = wgmma_desc_sw128(k_base + buf * Cfg::K_BYTES + (ksel[u] * DC + c) * FA_KCHUNK, 16, 1024);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<64>(s, qd + 2 * k, kd + 2 * k, (u > 0 || c > 0 || k > 0) ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    if ((tid & 127) == 0) mbar_arrive(&empty_k[buf]);
    // without a producer the single buffer is refilled as soon as both warpgroups are done with it
    if (!PRODUCER && tid == 0 && t + 1 < n_tiles) {
      mbar_wait(&empty_k[buf], ph);
      load_k(t + 1);
    }

    // ---- online softmax (log2 domain); keys >= Lk score -inf. The mask test is compiled out of the VAE, which has no
    // masked keys: its per-element branches between S and the softmax made the VAE at B = 8, L = 4096 take 750 instead
    // of 630 us (H100 80GB HBM3, 700 W power limit). The test is one branch per tile, not one per score, and on full
    // unmasked tiles the head-64 bf16 entry leaves S unscaled: softmax_step folds the scale into the FMA in front of
    // each exponential. The parity mode and the VAE scale S first, as a separate rounding, so their arithmetic is
    // unchanged.
    const int kv0 = t * FA_BN;
    const bool tail = D == 64 && ((kb != nullptr) || (kv0 + FA_BN > p.Lk));
    const bool fold = D == 64 && NSPLIT == 1 && !tail;
    if (tail) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int kv = kv0 + 8 * j + 2 * t4 + e;
          const float bias = kv < p.Lk ? (kb ? __ldg(kb + kv) * LOG2E : 0.f) : -INFINITY;
          s[4 * j + e] = fmaf(s[4 * j + e], sc, bias);
          s[4 * j + 2 + e] = fmaf(s[4 * j + 2 + e], sc, bias);
        }
      }
    } else if (!fold) {
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] = fmaf(s[i], sc, 0.f);
    }
    float corr[2];
    // the parity mode keeps every exponential on ex2.approx (it is held to 1e-3 of fp32), and so does the VAE
    softmax_step<(D == 64 && NSPLIT == 1) ? FA_POLY_EVERY : 0>(s, fold ? sc : 1.f, m_run, l_run, corr);
#pragma unroll
    for (int n = 0; n < NV; ++n) rescale_rows(o[n], corr);
    uint32_t pa[NSPLIT][4][4];
    pack_p(pa[0], s);
    if constexpr (NSPLIT == 2) pack_p<true>(pa[1], s);

    // ---- O += P V  (V rows = keys: MN-major B operand, 16 keys = 2048 bytes per k-step)
    mbar_wait(&full_v[buf], ph);
#pragma unroll
    for (int n = 0; n < NV; ++n) fence_regs(o[n]);
    wgmma_fence();
#pragma unroll
    for (int u = 0; u < NT; ++u) {
      const int ps = (NSPLIT == 2 && u == 1) ? NSPLIT - 1 : 0;   // P lo only in the lo*hi term
#pragma unroll
      for (int n = 0; n < NV; ++n) {
        const uint64_t vd = wgmma_desc_sw128(v_base + buf * Cfg::V_BYTES + (ksel[u] * NV + n) * FA_KCHUNK, 1024, 1024);
#pragma unroll
        for (int kk = 0; kk < FA_BN / 16; ++kk) wgmma_rs_n64_tb(o[n], pa[ps][kk], vd + ((kk * 2048) >> 4), 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int n = 0; n < NV; ++n) fence_regs(o[n]);
    if ((tid & 127) == 0) mbar_arrive(&empty_v[buf]);
    if (!PRODUCER && tid == 0 && t + 1 < n_tiles) {
      mbar_wait(&empty_v[buf], ph);
      load_v(t + 1);
    }
  }

  // ---- finalize: O / l -> bf16 (hi/lo)
  float inv[2];
  softmax_inv(l_run, inv);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * h;
    if (q >= p.Lq) continue;
    __nv_bfloat16* op = p.out + (static_cast<long long>(b) * p.Lq + q) * p.ld_o + vo_col + 2 * t4;
#pragma unroll
    for (int n = 0; n < NV; ++n)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float y0 = o[n][4 * j + 2 * h] * inv[h], y1 = o[n][4 * j + 2 * h + 1] * inv[h];
        *reinterpret_cast<uint32_t*>(op + 64 * n + 8 * j) = pack_bf16(y0, y1);
        if (p.split_off > 0)
          *reinterpret_cast<uint32_t*>(op + p.split_off + 64 * n + 8 * j) = pack_bf16_lo(y0, y1);
      }
  }
}

// Q in boxes of 128 rows, K / V in boxes of 64 keys; grid (ceil(Lq / 128), ny column slices, batch).
template <int D, int DV, int NSPLIT, int NBUF>
static int launch_flash(const void* q, long long ld_q, const void* k, long long ld_k, const void* v, long long ld_v,
                        int batch, int ny, const AttnParams& p, const char* what, void* stream) {
  constexpr int smem_bytes = FlashCfg<D, DV, NSPLIT, NBUF>::SMEM_BYTES;
  CUtensorMap qm, km, vm;
  int rc = encode_tmap_rows_bf16(&qm, q, ld_q, p.Lq, batch, FA_BM);
  if (!rc) rc = encode_tmap_rows_bf16(&km, k, ld_k, p.Lk, batch, FA_BN);
  if (!rc) rc = encode_tmap_rows_bf16(&vm, v, ld_v, p.Lk, batch, FA_BN);
  if (!rc) rc = set_max_dynamic_smem<flash_attention_kernel<D, DV, NSPLIT, NBUF>>(smem_bytes, what);
  if (rc) return rc;
  dim3 grid((p.Lq + FA_BM - 1) / FA_BM, ny, batch);
  flash_attention_kernel<D, DV, NSPLIT, NBUF>
      <<<grid, fa_threads(NBUF), smem_bytes, reinterpret_cast<cudaStream_t>(stream)>>>(qm, km, vm, p);
  return check_launch(what);
}

}  // namespace tng

using namespace tng;

extern "C" int tng_attention(const tng_attn_desc* d, void* stream) {
  if (!d || !d->q || !d->k || !d->v || !d->out) return set_error(TNG_EINVAL, "attention: null argument");
  if (d->nsplit != 1 && d->nsplit != 2) return set_error(TNG_EINVAL, "attention: nsplit=%d", d->nsplit);
  if (d->batch <= 0 || d->heads <= 0 || d->Lq <= 0 || d->Lk <= 0) return set_error(TNG_EINVAL, "attention: bad sizes");
  if (d->scale <= 0.f) return set_error(TNG_EINVAL, "attention: scale must be positive");
  if (d->ld_o % 8 || d->split_off % 8 || (reinterpret_cast<uintptr_t>(d->out) & 15))
    return set_error(TNG_EINVAL, "attention: output must allow 16-byte stores");
  AttnParams p;
  p.Lq = d->Lq; p.Lk = d->Lk;
  p.q_col0 = d->q_col0; p.q_lo_off = d->q_lo_off;
  p.k_col0 = d->k_col0; p.k_lo_off = d->k_lo_off;
  p.v_col0 = d->v_col0; p.v_lo_off = d->v_lo_off;
  p.kbias = d->kbias;
  p.out = reinterpret_cast<__nv_bfloat16*>(d->out);
  p.ld_o = d->ld_o; p.split_off = d->split_off;
  p.scale_log2e = d->scale * 1.4426950408889634f;
  if (d->nsplit == 2)
    return launch_flash<64, 64, 2, 3>(d->q, d->ld_q, d->k, d->ld_k, d->v, d->ld_v, d->batch, d->heads, p, "attention",
                                      stream);
  return launch_flash<64, 64, 1, 3>(d->q, d->ld_q, d->k, d->ld_k, d->v, d->ld_v, d->batch, d->heads, p, "attention",
                                    stream);
}

extern "C" int tng_attention_wide(const void* q, int64_t ld_q, int32_t q_col0, const void* k, int64_t ld_k, int32_t k_col0,
                                  const void* v, int64_t ld_v, int32_t v_col0, void* out, int64_t ld_o, int32_t batch,
                                  int32_t L, int32_t dim, float scale, void* stream) {
  if (!q || !k || !v || !out || batch <= 0 || L <= 0) return set_error(TNG_EINVAL, "attention_wide: bad argument");
  if (dim != 512) return set_error(TNG_EINVAL, "attention_wide: head width %d unsupported (512 only)", dim);
  if (L % FA_BM != 0) return set_error(TNG_EINVAL, "attention_wide: L = %d must be a multiple of %d", L, FA_BM);
  if (scale <= 0.f) return set_error(TNG_EINVAL, "attention_wide: scale must be positive");
  if (ld_o % 8 || (reinterpret_cast<uintptr_t>(out) & 15)) return set_error(TNG_EINVAL, "attention_wide: output must allow 16-byte stores");
  AttnParams p{};   // no key mask, no lo operands or output
  p.Lq = L; p.Lk = L;
  p.q_col0 = q_col0; p.k_col0 = k_col0; p.v_col0 = v_col0;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ld_o = ld_o;
  p.scale_log2e = scale * 1.4426950408889634f;
  // blockIdx.y = the two 256-column halves of V / O
  return launch_flash<512, 256, 1, 1>(q, ld_q, k, ld_k, v, ld_v, batch, 2, p, "attention_wide", stream);
}
