// attention_wide.cu — wgmma flash attention for ONE head of width 512: the AudioLDM VAE AttnBlock
// (audioldm/variational_autoencoder/modules.py:204-230: softmax(q k^T / sqrt(C)) v over the H*W positions of an image,
// C = 512, 4096 positions for a 10 s clip, 12288 for 30 s). The [HW, HW] score matrix never leaves the SM.
//
// One CTA = 128 query rows of one image x ONE HALF (256 columns) of the value / output width; grid (HW / 128, 2, batch).
//   smem  : Q [128 x 512] bf16 as 8 SWIZZLE_128B chunks (128 KB, loaded once), one K sub-tile [64 keys x 512] (64 KB),
//           one V sub-tile [64 keys x 256] (32 KB)  -> 224 KB, which is why K / V are single-buffered;
//   regs  : 256 threads = two warpgroups, warpgroup g owns query rows [64g, 64g + 64): S [64 x 64] fp32 (32 registers),
//           P as the bf16 A operand (16), O [64 x 256] fp32 (128).
// Per 64-key sub-tile g:  S = sum over the 8 head-dim chunks of Q_c K_c^T (32 wgmma m64n64k16)  ->  online softmax in
// registers  ->  O += P V (register-A wgmma, V consumed as an MN-major B operand, 64 output columns per instruction).
// K_{g+1} is requested as soon as both warpgroups have finished Q K_g^T and V_{g+1} when they have finished P V_g.
// Both halves recompute S (the score FLOPs double; they are 1/5 of a decoder that is itself < 1 % of a 200-step
// generation) so that the O accumulator fits the registers. bf16 operands only: the parity mode (hi/lo split) keeps the
// GEMM -> softmax -> GEMM formulation.
#include "tng_ptx.cuh"
#include "tng_internal.h"

namespace tng {

constexpr int AW_BM = 128;                 // queries per CTA
constexpr int AW_SUB = 64;                 // keys per sub-tile
constexpr int AW_D = 512;                  // head width
constexpr int AW_DV = 256;                 // value / output columns per CTA
constexpr int AW_QCH = AW_BM * 128;        // one [128][64] bf16 chunk = 16 KB
constexpr int AW_KCH = AW_SUB * 128;       // one [64][64] bf16 chunk = 8 KB
constexpr int AW_Q_BYTES = (AW_D / 64) * AW_QCH;       // 128 KB
constexpr int AW_K_BYTES = (AW_D / 64) * AW_KCH;       // 64 KB
constexpr int AW_V_BYTES = (AW_DV / 64) * AW_KCH;      // 32 KB
constexpr int AW_SMEM = AW_Q_BYTES + AW_K_BYTES + AW_V_BYTES + 128;
constexpr int AW_THREADS = 256;

struct AttnWideParams {
  int L;
  int q_col0, k_col0, v_col0;
  __nv_bfloat16* out;
  long long ld_o;
  float scale_log2e;
};

__global__ void __launch_bounds__(AW_THREADS, 1)
attention_wide_kernel(const __grid_constant__ CUtensorMap qmap, const __grid_constant__ CUtensorMap kmap,
                      const __grid_constant__ CUtensorMap vmap, const __grid_constant__ AttnWideParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + AW_Q_BYTES;
  uint8_t* sV = sK + AW_K_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + AW_V_BYTES);
  uint64_t* bar_q = bars;        // Q landed
  uint64_t* full_k = bars + 1;   // K sub-tile landed
  uint64_t* full_v = bars + 2;   // V sub-tile landed
  uint64_t* empty_k = bars + 3;  // both warpgroups are done with the K sub-tile
  uint64_t* empty_v = bars + 4;  // ... with the V sub-tile

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int wg = warp >> 2;
  const int q0 = blockIdx.x * AW_BM;
  const int half = blockIdx.y;
  const int b = blockIdx.z;
  const int n_sub = p.L / AW_SUB;

  auto load_k = [&](int g) {
    mbar_arrive_expect_tx(full_k, AW_K_BYTES);
#pragma unroll
    for (int c = 0; c < AW_D / 64; ++c) tma_load_3d(sK + c * AW_KCH, &kmap, full_k, p.k_col0 + 64 * c, g * AW_SUB, b);
  };
  auto load_v = [&](int g) {
    mbar_arrive_expect_tx(full_v, AW_V_BYTES);
#pragma unroll
    for (int c = 0; c < AW_DV / 64; ++c)
      tma_load_3d(sV + c * AW_KCH, &vmap, full_v, p.v_col0 + half * AW_DV + 64 * c, g * AW_SUB, b);
  };

  if (tid == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();   // SWIZZLE_128B tiles need a 1024-byte aligned base
    tma_prefetch_desc(&qmap);
    tma_prefetch_desc(&kmap);
    tma_prefetch_desc(&vmap);
    mbar_init(bar_q, 1);
    mbar_init(full_k, 1);
    mbar_init(full_v, 1);
    mbar_init(empty_k, 2);
    mbar_init(empty_v, 2);
    fence_mbar_init();
    mbar_arrive_expect_tx(bar_q, AW_Q_BYTES);
#pragma unroll
    for (int c = 0; c < AW_D / 64; ++c) tma_load_3d(sQ + c * AW_QCH, &qmap, bar_q, p.q_col0 + 64 * c, q0, b);
    load_k(0);
    load_v(0);
  }
  __syncthreads();

  const uint32_t q_base = smem_u32(sQ) + wg * (64 * 128);   // this warpgroup's 64 query rows
  const uint32_t k_base = smem_u32(sK), v_base = smem_u32(sV);
  const float sc = p.scale_log2e;
  // this thread holds rows (lane >> 2) and (lane >> 2) + 8 of its warp's 16 rows
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
  float o[AW_DV / 64][32];
#pragma unroll
  for (int n = 0; n < AW_DV / 64; ++n)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[n][i] = 0.f;

  mbar_wait(bar_q, 0);
  for (int g = 0; g < n_sub; ++g) {
    const uint32_t ph = g & 1;
    // ---- S_g = Q K_g^T over the 512-wide head: 8 chunks x 4 K-steps of 16
    float s[32];
    mbar_wait(full_k, ph);
    fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < AW_D / 64; ++c) {
      const uint64_t qd = wgmma_desc_sw128(q_base + c * AW_QCH, 16, 1024);
      const uint64_t kd = wgmma_desc_sw128(k_base + c * AW_KCH, 16, 1024);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss<64>(s, qd + 2 * k, kd + 2 * k, (c > 0 || k > 0) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    if ((tid & 127) == 0) mbar_arrive(empty_k);
    if (tid == 0 && g + 1 < n_sub) {
      mbar_wait(empty_k, ph);
      load_k(g + 1);
    }

    // ---- online softmax (log2 domain)
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] *= sc;
    float corr[2];
    softmax_step(s, m_run, l_run, corr);
#pragma unroll
    for (int n = 0; n < AW_DV / 64; ++n) rescale_rows(o[n], corr);
    uint32_t pa[4][4];
    pack_p(pa, s);

    // ---- O (+)= P_g V_g: 16 keys per k-step (16 x 128 B rows of each 64-column V chunk)
    mbar_wait(full_v, ph);
#pragma unroll
    for (int n = 0; n < AW_DV / 64; ++n) fence_regs(o[n]);
    wgmma_fence();
#pragma unroll
    for (int n = 0; n < AW_DV / 64; ++n) {
      const uint64_t vd = wgmma_desc_sw128(v_base + n * AW_KCH, 1024, 1024);
#pragma unroll
      for (int kk = 0; kk < AW_SUB / 16; ++kk) wgmma_rs_n64_tb(o[n], pa[kk], vd + ((kk * 2048) >> 4), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int n = 0; n < AW_DV / 64; ++n) fence_regs(o[n]);
    if ((tid & 127) == 0) mbar_arrive(empty_v);
    if (tid == 0 && g + 1 < n_sub) {
      mbar_wait(empty_v, ph);
      load_v(g + 1);
    }
  }

  // ---- finalize: O / l -> bf16
  const int t4 = lane & 3;
  float inv[2];
  softmax_inv(l_run, inv);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * h;
    __nv_bfloat16* op = p.out + (static_cast<long long>(b) * p.L + q) * p.ld_o + half * AW_DV + 2 * t4;
#pragma unroll
    for (int n = 0; n < AW_DV / 64; ++n)
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint32_t*>(op + 64 * n + 8 * j) =
            pack_bf16(o[n][4 * j + 2 * h] * inv[h], o[n][4 * j + 2 * h + 1] * inv[h]);
  }
}

}  // namespace tng

using namespace tng;

extern "C" int tng_attention_wide(const void* q, int64_t ld_q, int32_t q_col0, const void* k, int64_t ld_k, int32_t k_col0,
                                  const void* v, int64_t ld_v, int32_t v_col0, void* out, int64_t ld_o, int32_t batch,
                                  int32_t L, int32_t dim, float scale, void* stream) {
  if (!q || !k || !v || !out || batch <= 0 || L <= 0) return set_error(TNG_EINVAL, "attention_wide: bad argument");
  if (dim != AW_D) return set_error(TNG_EINVAL, "attention_wide: head width %d unsupported (512 only)", dim);
  if (L % AW_BM != 0) return set_error(TNG_EINVAL, "attention_wide: L = %d must be a multiple of %d", L, AW_BM);
  if (scale <= 0.f) return set_error(TNG_EINVAL, "attention_wide: scale must be positive");
  if (ld_o % 8 || (reinterpret_cast<uintptr_t>(out) & 15)) return set_error(TNG_EINVAL, "attention_wide: output must allow 16-byte stores");
  AttnWideParams p;
  p.L = L; p.q_col0 = q_col0; p.k_col0 = k_col0; p.v_col0 = v_col0;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ld_o = ld_o;
  p.scale_log2e = scale * 1.4426950408889634f;
  CUtensorMap qm, km, vm;
  int rc = encode_tmap_rows_bf16(&qm, q, ld_q, L, batch, AW_BM);
  if (!rc) rc = encode_tmap_rows_bf16(&km, k, ld_k, L, batch, AW_SUB);
  if (!rc) rc = encode_tmap_rows_bf16(&vm, v, ld_v, L, batch, AW_SUB);
  if (!rc) rc = set_max_dynamic_smem<attention_wide_kernel>(AW_SMEM, "attention_wide");
  if (rc) return rc;
  dim3 grid(L / AW_BM, AW_D / AW_DV, batch);
  attention_wide_kernel<<<grid, AW_THREADS, AW_SMEM, reinterpret_cast<cudaStream_t>(stream)>>>(qm, km, vm, p);
  return check_launch("attention_wide");
}
