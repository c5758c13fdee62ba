// attention_tc.cu — wgmma flash attention for head width 64 (UNet self- and cross-attention), sm_90a.
//
// One CTA = 128 query rows of one (batch, head), 256 threads: warpgroup g owns query rows [64g, 64g + 64). Q / K / V
// arrive as TMA SWIZZLE_128B tiles (K / V in tiles of 64 keys, NB buffers deep, refilled by thread 0). Per key tile:
// S = Q K^T (wgmma m64n64k16, both operands K-major in shared memory) -> fp32 online softmax in registers (the four
// lanes that share a row combine their maxima / sums by shuffles) -> O += P V with P taken straight from registers as
// the A operand (the accumulator layout of S is the A-fragment layout) and V consumed as an MN-major B operand (no
// transpose). Two CTAs per SM in perf mode.
// NSPLIT = 2 is the parity mode: every operand carries its bf16 rounding residual and each product is evaluated as
// hi*hi + lo*hi + hi*lo, which restores ~fp32 accuracy on the bf16 tensor cores (1 CTA / SM).
#include "tng_ptx.cuh"
#include "tng_internal.h"
#include <stdlib.h>

namespace tng {

constexpr int AT_BM = 128;   // queries per CTA
constexpr int AT_BN = 64;    // keys per tile
constexpr int AT_D = 64;     // head width
constexpr int AT_QCHUNK = AT_BM * 128;   // one [128][64] bf16 swizzled chunk = 16 KB
constexpr int AT_KCHUNK = AT_BN * 128;   // one [64][64] bf16 swizzled chunk = 8 KB
constexpr int AT_NB = 3;                 // K / V tile buffers
constexpr int AT_THREADS = 256;

struct AttnParams {
  int Lq, Lk, heads;
  int q_col0, q_lo_off, k_col0, k_lo_off, v_col0, v_lo_off;
  const float* kbias;
  __nv_bfloat16* out;
  long long ld_o;
  int split_off;
  float scale_log2e;  // scale * log2(e)
};

template <int NSPLIT>
struct AttnCfg {
  static constexpr int Q_BYTES = NSPLIT * AT_QCHUNK;
  static constexpr int KV_BYTES = NSPLIT * AT_KCHUNK;     // each of K and V per buffer
  static constexpr int SMEM_BYTES = Q_BYTES + AT_NB * 2 * KV_BYTES + 128;
};

template <int NSPLIT>
__global__ void __launch_bounds__(AT_THREADS, (NSPLIT == 1) ? 2 : 1)
attention_kernel(const __grid_constant__ CUtensorMap qmap, const __grid_constant__ CUtensorMap kmap,
                 const __grid_constant__ CUtensorMap vmap, const __grid_constant__ AttnParams p) {
  using Cfg = AttnCfg<NSPLIT>;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::Q_BYTES;                 // [NB][KV_BYTES]
  uint8_t* sV = sK + AT_NB * Cfg::KV_BYTES;        // [NB][KV_BYTES]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + AT_NB * Cfg::KV_BYTES);
  uint64_t* bar_q = bars;                          // [1]
  uint64_t* full_k = bars + 1;                     // [NB] K tile landed
  uint64_t* full_v = bars + 1 + AT_NB;             // [NB] V tile landed
  uint64_t* empty_k = bars + 1 + 2 * AT_NB;        // [NB] both warpgroups are done with the K buffer
  uint64_t* empty_v = bars + 1 + 3 * AT_NB;        // [NB] ... with the V buffer

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int wg = warp >> 2;
  const int q0 = blockIdx.x * AT_BM;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int n_tiles = (p.Lk + AT_BN - 1) / AT_BN;

  auto load_k = [&](int t) {
    const int buf = t % AT_NB;
    mbar_arrive_expect_tx(&full_k[buf], Cfg::KV_BYTES);
#pragma unroll
    for (int s = 0; s < NSPLIT; ++s)
      tma_load_3d(sK + buf * Cfg::KV_BYTES + s * AT_KCHUNK, &kmap, &full_k[buf], p.k_col0 + s * p.k_lo_off + head * AT_D,
                  t * AT_BN, b);
  };
  auto load_v = [&](int t) {
    const int buf = t % AT_NB;
    mbar_arrive_expect_tx(&full_v[buf], Cfg::KV_BYTES);
#pragma unroll
    for (int s = 0; s < NSPLIT; ++s)
      tma_load_3d(sV + buf * Cfg::KV_BYTES + s * AT_KCHUNK, &vmap, &full_v[buf], p.v_col0 + s * p.v_lo_off + head * AT_D,
                  t * AT_BN, b);
  };

  if (tid == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();   // SWIZZLE_128B tiles need a 1024-byte aligned base
    tma_prefetch_desc(&qmap);
    tma_prefetch_desc(&kmap);
    tma_prefetch_desc(&vmap);
    mbar_init(bar_q, 1);
    for (int i = 0; i < AT_NB; ++i) {
      mbar_init(&full_k[i], 1);
      mbar_init(&full_v[i], 1);
      mbar_init(&empty_k[i], 2);
      mbar_init(&empty_v[i], 2);
    }
    fence_mbar_init();
    mbar_arrive_expect_tx(bar_q, Cfg::Q_BYTES);
#pragma unroll
    for (int s = 0; s < NSPLIT; ++s)
      tma_load_3d(sQ + s * AT_QCHUNK, &qmap, bar_q, p.q_col0 + s * p.q_lo_off + head * AT_D, q0, b);
    for (int t = 0; t < AT_NB && t < n_tiles; ++t) { load_k(t); load_v(t); }
  }
  __syncthreads();

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
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;

  mbar_wait(bar_q, 0);
  for (int t = 0; t < n_tiles; ++t) {
    const int buf = t % AT_NB;
    const uint32_t ph = (t / AT_NB) & 1;
    // refill the buffers of tile t - 1 (released by both warpgroups at the end of that tile) with tile t - 1 + NB
    if (tid == 0 && t >= 1 && t - 1 + AT_NB < n_tiles) {
      const int pb = (t - 1) % AT_NB;
      const uint32_t pph = ((t - 1) / AT_NB) & 1;
      mbar_wait(&empty_k[pb], pph);
      load_k(t - 1 + AT_NB);
      mbar_wait(&empty_v[pb], pph);
      load_v(t - 1 + AT_NB);
    }
    // ---- S = Q K^T over the 64 keys of tile t
    float s[32];
    mbar_wait(&full_k[buf], ph);
    fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int u = 0; u < NT; ++u) {
      const uint64_t qd = wgmma_desc_sw128(q_base + qsel[u] * AT_QCHUNK, 16, 1024);
      const uint64_t kd = wgmma_desc_sw128(k_base + buf * Cfg::KV_BYTES + ksel[u] * AT_KCHUNK, 16, 1024);
#pragma unroll
      for (int k = 0; k < AT_D / 16; ++k) wgmma_ss<64>(s, qd + 2 * k, kd + 2 * k, (u > 0 || k > 0) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    if ((tid & 127) == 0) mbar_arrive(&empty_k[buf]);

    // ---- online softmax (log2 domain); keys >= Lk score -inf
    const int kv0 = t * AT_BN;
    const bool tail = (kb != nullptr) || (kv0 + AT_BN > p.Lk);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float bias = 0.f;
        if (tail) {
          const int kv = kv0 + 8 * j + 2 * t4 + e;
          bias = kv < p.Lk ? (kb ? __ldg(kb + kv) * LOG2E : 0.f) : -INFINITY;
        }
        s[4 * j + e] = fmaf(s[4 * j + e], sc, bias);
        s[4 * j + 2 + e] = fmaf(s[4 * j + 2 + e], sc, bias);
      }
    }
    float corr[2];
    softmax_step(s, m_run, l_run, corr);
    rescale_rows(o, corr);
    uint32_t pa[NSPLIT][4][4];
    pack_p(pa[0], s);
    if constexpr (NSPLIT == 2) pack_p<true>(pa[1], s);

    // ---- O += P V  (V rows = keys: MN-major B operand, 16 keys = 2048 bytes per k-step)
    mbar_wait(&full_v[buf], ph);
    fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int u = 0; u < NT; ++u) {
      const int ps = (NSPLIT == 2 && u == 1) ? NSPLIT - 1 : 0;   // P lo only in the lo*hi term
      const uint64_t vd = wgmma_desc_sw128(v_base + buf * Cfg::KV_BYTES + ksel[u] * AT_KCHUNK, 1024, 1024);
#pragma unroll
      for (int kk = 0; kk < AT_BN / 16; ++kk) wgmma_rs_n64_tb(o, pa[ps][kk], vd + ((kk * 2048) >> 4), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    if ((tid & 127) == 0) mbar_arrive(&empty_v[buf]);
  }

  // ---- finalize: O / l -> bf16 (hi/lo)
  float inv[2];
  softmax_inv(l_run, inv);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * h;
    if (q >= p.Lq) continue;
    __nv_bfloat16* op = p.out + (static_cast<long long>(b) * p.Lq + q) * p.ld_o + head * AT_D + 2 * t4;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float y0 = o[4 * j + 2 * h] * inv[h], y1 = o[4 * j + 2 * h + 1] * inv[h];
      *reinterpret_cast<uint32_t*>(op + 8 * j) = pack_bf16(y0, y1);
      if (p.split_off > 0)
        *reinterpret_cast<uint32_t*>(op + p.split_off + 8 * j) = pack_bf16_lo(y0, y1);
    }
  }
}

template <int NSPLIT>
static int launch_attn(const tng_attn_desc* d, const CUtensorMap& qm, const CUtensorMap& km, const CUtensorMap& vm,
                       const AttnParams& p, cudaStream_t st) {
  const int rc = set_max_dynamic_smem<attention_kernel<NSPLIT>>(AttnCfg<NSPLIT>::SMEM_BYTES, "attention");
  if (rc) return rc;
  dim3 grid((d->Lq + AT_BM - 1) / AT_BM, d->heads, d->batch);
  attention_kernel<NSPLIT><<<grid, AT_THREADS, AttnCfg<NSPLIT>::SMEM_BYTES, st>>>(qm, km, vm, p);
  return check_launch("attention");
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
  p.Lq = d->Lq; p.Lk = d->Lk; p.heads = d->heads;
  p.q_col0 = d->q_col0; p.q_lo_off = d->q_lo_off;
  p.k_col0 = d->k_col0; p.k_lo_off = d->k_lo_off;
  p.v_col0 = d->v_col0; p.v_lo_off = d->v_lo_off;
  p.kbias = d->kbias;
  p.out = reinterpret_cast<__nv_bfloat16*>(d->out);
  p.ld_o = d->ld_o; p.split_off = d->split_off;
  p.scale_log2e = d->scale * 1.4426950408889634f;
  CUtensorMap qm, km, vm;
  int rc = encode_tmap_rows_bf16(&qm, d->q, d->ld_q, d->Lq, d->batch, AT_BM);
  if (!rc) rc = encode_tmap_rows_bf16(&km, d->k, d->ld_k, d->Lk, d->batch, AT_BN);
  if (!rc) rc = encode_tmap_rows_bf16(&vm, d->v, d->ld_v, d->Lk, d->batch, AT_BN);
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (d->nsplit == 2) return launch_attn<2>(d, qm, km, vm, p, st);
  return launch_attn<1>(d, qm, km, vm, p, st);
}
