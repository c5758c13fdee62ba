// latent_step.cu — the latent updates run between two UNet replays: the DDPM / DDIM step, the multistep DPM-Solver
// step, the UniPC predictor-corrector step and the latent blend of editing / inpainting. Each is fused with the CFG combine it reads and the packing of the
// next UNet input, in one HBM pass. The per-step scalars come from a host-computed coefficient row (device pointer, see
// tango_b200/schedulers.py); every product and sum is one IEEE round-to-nearest op in the reference's association
// order, so each update equals the reference's fp32 CPU arithmetic bit for bit.
#include "tng_ptx.cuh"
#include "tng_internal.h"

namespace tng {

// What the three updates share. mo: the model output, fp32 channels-last [(2)B, HW, ld_mo] (uncond half first under
// CFG), NULL when the update reads none; out: the new latent, fp32 NCHW [B, C, HW]; next_in: the next UNet input, bf16
// channels-last [(2)B, HW, ld_in] (duplicated for the CFG halves, hi/lo split at split_off when > 0).
struct LatentStep {
  const float* mo;
  long long ld_mo;
  int cfg;
  float guidance;
  const float* coef;
  float* out;
  __nv_bfloat16* next_in;
  long long ld_in;
  int split_off;
  long long B;
  int C;
  long long HW;
};

// Element nchw of the NCHW latent and its (b, c, hw) coordinates
struct LatentElem {
  long long nchw, b, hw;
  int c;
};

// The model output an update uses: u + guidance * (t - u) under CFG (models.py:246, no fma contraction)
__device__ __forceinline__ float guided_output(const LatentStep& p, const LatentElem& e) {
  const float u = p.mo[(e.b * p.HW + e.hw) * p.ld_mo + e.c];
  if (!p.cfg) return u;
  const float t = p.mo[((p.B + e.b) * p.HW + e.hw) * p.ld_mo + e.c];
  return __fadd_rn(u, __fmul_rn(p.guidance, __fsub_rn(t, u)));
}

__device__ __forceinline__ void store_next_input(const LatentStep& p, const LatentElem& e, float x) {
  store_bf16_split(p.next_in + (e.b * p.HW + e.hw) * p.ld_in + e.c, x, p.split_off);
  if (p.cfg) store_bf16_split(p.next_in + ((p.B + e.b) * p.HW + e.hw) * p.ld_in + e.c, x, p.split_off);
}

// DDPMScheduler.step (scheduling_ddpm.py:306-311) / DDIMScheduler.step (scheduling_ddim.py:303-313); with no model
// output the sample itself, which packs the loop's initial latents.
struct SchedStep {
  static constexpr int kCoefs = 10;
  const float* sample;
  const float* noise;
  __device__ float operator()(const LatentStep& p, const float* k, const LatentElem& e) const {
    const float c_x0_s = k[0], c_x0_m = k[1], c_prev_x0 = k[2], c_prev_s = k[3], c_noise = k[4];
    const float c_eps_s = k[5], c_eps_m = k[6], c_prev_eps = k[7], clip = k[8], c_x0_div = k[9];
    const float s = sample[e.nchw];
    if (!p.mo) return s;
    const float v = guided_output(p, e);
    float x0 = __fdiv_rn(__fadd_rn(__fmul_rn(c_x0_s, s), __fmul_rn(c_x0_m, v)), c_x0_div);
    if (clip > 0.f) x0 = fminf(fmaxf(x0, -clip), clip);
    float out = __fadd_rn(__fmul_rn(c_prev_x0, x0), __fmul_rn(c_prev_s, s));
    if (c_prev_eps != 0.f) {
      const float eps = __fadd_rn(__fmul_rn(c_eps_s, s), __fmul_rn(c_eps_m, v));
      out = __fadd_rn(out, __fmul_rn(c_prev_eps, eps));
    }
    if (noise && c_noise != 0.f) out = __fadd_rn(out, __fmul_rn(c_noise, noise[e.nchw]));
    return out;
  }
};

// DPMSolverMultistepScheduler.step: convert_model_output (scheduling_dpmsolver_multistep.py:243-281, all six
// (algorithm, prediction) pairs) written to the history slot m0, then the update of `order` from m0, m1, m2.
struct DpmStep {
  static constexpr int kCoefs = 11;
  const float* sample;
  int order;
  float* m0_out;
  const float* m1_in;
  const float* m2_in;
  __device__ float operator()(const LatentStep& p, const float* k, const LatentElem& e) const {
    const float c_a = k[0], c_b = k[1], c_d = k[2], c_s = k[3], c_0 = k[4], c_1 = k[5], c_2 = k[6];
    const float inv_r0 = k[7], inv_r1 = k[8], w_r = k[9], inv_r01 = k[10];
    const float s = sample[e.nchw];
    const float v = guided_output(p, e);
    const float m0 = __fdiv_rn(__fadd_rn(__fmul_rn(c_a, s), __fmul_rn(c_b, v)), c_d);
    m0_out[e.nchw] = m0;
    // first-order update (:305-313); the higher orders add their D1 / D2 terms in the reference's order (:336-427)
    float x = __fsub_rn(__fmul_rn(c_s, s), __fmul_rn(c_0, m0));
    if (order == 2) {
      const float d1 = __fmul_rn(inv_r0, __fsub_rn(m0, m1_in[e.nchw]));
      x = __fadd_rn(x, __fmul_rn(c_1, d1));
    } else if (order == 3) {
      const float m1 = m1_in[e.nchw];
      const float d1_0 = __fmul_rn(inv_r0, __fsub_rn(m0, m1));
      const float d1_1 = __fmul_rn(inv_r1, __fsub_rn(m1, m2_in[e.nchw]));
      const float dd = __fsub_rn(d1_0, d1_1);
      const float d1 = __fadd_rn(d1_0, __fmul_rn(w_r, dd));
      const float d2 = __fmul_rn(inv_r01, dd);
      x = __fsub_rn(__fadd_rn(x, __fmul_rn(c_1, d1)), __fmul_rn(c_2, d2));
    }
    return x;
  }
};

// UniPCMultistepScheduler.step (scheduling_unipc_multistep.py:490-572): convert_model_output (:225-278) from the
// uncorrected sample, written to the history slot m_out; the UniC corrector of order p (:384-488; p = 0: none) from
// last, m1 = m_{i-1} and the older slots, written back to last; then the UniP predictor of order q (:279-382) from
// the corrected sample, m_out, m1 and m2. The two-term einsum of the fork is fma(rho_1, D1_1, rho_0 * D1_0).
struct UniPcStep {
  static constexpr int kCoefs = 18;
  const float* sample;
  int p, q;
  float* m_out;
  const float* m1_in;
  const float* m2_in;
  const float* m3_in;
  float* last;
  __device__ float operator()(const LatentStep& pr, const float* k, const LatentElem& e) const {
    const float s = sample[e.nchw];
    const float v = guided_output(pr, e);
    const float m = __fdiv_rn(__fadd_rn(__fmul_rn(k[0], s), __fmul_rn(k[1], v)), k[2]);
    m_out[e.nchw] = m;
    float x = s;
    if (p > 0) {
      // x_t_ - c_b * (corr_res + rho_last * (m - m_{i-1})), x_t_ = c_x * last - c_m * m_{i-1}; corr_res = 0 for p = 1
      const float m1 = m1_in[e.nchw];
      float corr = 0.f;
      if (p >= 2) {
        const float d0 = __fdiv_rn(__fsub_rn(m2_in[e.nchw], m1), k[6]);
        corr = __fmul_rn(k[8], d0);
        if (p == 3) corr = __fmaf_rn(k[9], __fdiv_rn(__fsub_rn(m3_in[e.nchw], m1), k[7]), corr);
      }
      const float sum = __fadd_rn(corr, __fmul_rn(k[10], __fsub_rn(m, m1)));
      x = __fsub_rn(__fsub_rn(__fmul_rn(k[3], last[e.nchw]), __fmul_rn(k[4], m1)), __fmul_rn(k[5], sum));
    }
    if (last) last[e.nchw] = x;
    // x_t_ - c_b * pred_res, x_t_ = c_x * x - c_m * m; pred_res = 0 for q = 1
    float res = 0.f;
    if (q >= 2) {
      const float d0 = __fdiv_rn(__fsub_rn(m1_in[e.nchw], m), k[14]);
      res = __fmul_rn(k[16], d0);
      if (q == 3) res = __fmaf_rn(k[17], __fdiv_rn(__fsub_rn(m2_in[e.nchw], m), k[15]), res);
    }
    return __fsub_rn(__fsub_rn(__fmul_rn(k[11], x), __fmul_rn(k[12], m)), __fmul_rn(k[13], res));
  }
};

// The schedulers' add_noise (scheduling_ddpm.py:351-372) and, under a mask, the legacy-inpaint blend
// (pipeline_stable_diffusion_inpaint_legacy.py:692-709).
struct LatentBlend {
  static constexpr int kCoefs = 2;
  const float* x0;
  const float* noise;
  const float* mask;
  long long mask_bstride;
  const float* sample;
  __device__ float operator()(const LatentStep&, const float* k, const LatentElem& e) const {
    const float sqrt_a = k[0], sqrt_1ma = k[1];
    // add_noise: sqrt_alpha_prod * original_samples + sqrt_one_minus_alpha_prod * noise
    float out = __fmul_rn(sqrt_a, x0[e.nchw]);
    if (noise) out = __fadd_rn(out, __fmul_rn(sqrt_1ma, noise[e.nchw]));
    if (mask) {
      // (init_latents_proper * mask) + (latents * (1 - mask))
      const float m = mask[e.b * mask_bstride + e.hw];
      out = __fadd_rn(__fmul_rn(out, m), __fmul_rn(sample[e.nchw], __fsub_rn(1.0f, m)));
    }
    return out;
  }
};

// One thread per latent element, walked channels-last (c fastest, then hw, then b): a warp's model-output reads and
// bf16 input writes are contiguous, and its NCHW reads and writes are C runs of 32 / C consecutive pixels whose lines
// the warps of the neighbouring pixels share. At the UNet's C = 8 this is faster than an NCHW walk for all three
// updates.
template <class Update>
__global__ void __launch_bounds__(256) latent_step_kernel(const LatentStep p, const Update up) {
  float k[Update::kCoefs];
#pragma unroll
  for (int i = 0; i < Update::kCoefs; ++i) k[i] = p.coef[i];
  const long long total = p.B * p.C * p.HW;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % p.C);
    const long long hw = (i / p.C) % p.HW;
    const long long b = i / (p.C * p.HW);
    const LatentElem e{(b * p.C + c) * p.HW + hw, b, hw, c};
    const float x = up(p, k, e);
    if (p.out) p.out[e.nchw] = x;
    if (p.next_in) store_next_input(p, e, x);
  }
}

// The checks the three entry points share, every one before any CUDA call, then the launch over the [B, C, HW] shape;
// `pointers_ok`: the entry point's own required pointers are all non-null.
template <class Update>
int launch_latent_step(const char* what, bool pointers_ok, LatentStep p, int64_t B, int64_t C, int64_t HW,
                       const Update& up, void* stream) {
  if (!pointers_ok || !p.coef || (!p.out && !p.next_in)) return set_error(TNG_EINVAL, "%s: null argument", what);
  if (B < 1 || C < 1 || C > INT32_MAX || HW < 1)
    return set_error(TNG_EINVAL, "%s: bad shape B=%lld C=%lld HW=%lld", what, (long long)B, (long long)C,
                     (long long)HW);
  if (p.mo && p.ld_mo < C) return set_error(TNG_EINVAL, "%s: ld_mo %lld < C %lld", what, p.ld_mo, (long long)C);
  if (p.next_in && p.split_off != 0 && p.split_off < C)
    return set_error(TNG_EINVAL, "%s: split_off %d is neither 0 nor >= C %lld", what, p.split_off, (long long)C);
  if (p.next_in && p.ld_in < C + p.split_off)
    return set_error(TNG_EINVAL, "%s: ld_in %lld < C %lld + split_off %d", what, p.ld_in, (long long)C, p.split_off);
  p.B = B;
  p.C = static_cast<int>(C);
  p.HW = HW;
  latent_step_kernel<Update><<<grid_for(B * C * HW), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, up);
  return check_launch(what);
}

}  // namespace tng

using namespace tng;

extern "C" int tng_sched_step(const float* model_out, int64_t ld_mo, int32_t cfg, float guidance, const float* sample,
                              const float* noise, const float* coef, float* prev, void* next_in, int64_t ld_in,
                              int32_t split_off, int64_t B, int64_t C, int64_t HW, void* stream) {
  const LatentStep p{model_out, ld_mo, cfg, guidance, coef, prev, static_cast<__nv_bfloat16*>(next_in), ld_in,
                     split_off};
  return launch_latent_step("sched_step", sample != nullptr, p, B, C, HW, SchedStep{sample, noise}, stream);
}

extern "C" int tng_dpm_step(const float* model_out, int64_t ld_mo, int32_t cfg, float guidance, const float* sample,
                            const float* coef, int32_t order, float* m0, const float* m1, const float* m2, float* prev,
                            void* next_in, int64_t ld_in, int32_t split_off, int64_t B, int64_t C, int64_t HW,
                            void* stream) {
  if (order < 1 || order > 3) return set_error(TNG_EINVAL, "dpm_step: order %d is not 1, 2 or 3", order);
  if ((order >= 2 && !m1) || (order == 3 && !m2)) return set_error(TNG_EINVAL, "dpm_step: order %d needs its history", order);
  const LatentStep p{model_out, ld_mo, cfg, guidance, coef, prev, static_cast<__nv_bfloat16*>(next_in), ld_in,
                     split_off};
  return launch_latent_step("dpm_step", model_out && sample && m0, p, B, C, HW, DpmStep{sample, order, m0, m1, m2},
                            stream);
}

extern "C" int tng_unipc_step(const float* model_out, int64_t ld_mo, int32_t cfg, float guidance, const float* sample,
                              const float* coef, int32_t corrector_order, int32_t predictor_order, float* m_cur,
                              const float* m_prev1, const float* m_prev2, const float* m_prev3, float* last,
                              float* prev, void* next_in, int64_t ld_in, int32_t split_off, int64_t B, int64_t C,
                              int64_t HW, void* stream) {
  const int p = corrector_order, q = predictor_order;
  if (p < 0 || p > 3) return set_error(TNG_EINVAL, "unipc_step: corrector order %d is not 0, 1, 2 or 3", p);
  if (q < 1 || q > 3) return set_error(TNG_EINVAL, "unipc_step: predictor order %d is not 1, 2 or 3", q);
  // the corrector of order p reads m_{i-1} .. m_{i-p}, the predictor of order q m_{i-1} .. m_{i-q+1}
  const int depth = p > q - 1 ? p : q - 1;
  const float* hist[3] = {m_prev1, m_prev2, m_prev3};
  for (int j = 0; j < depth; ++j) {
    if (!hist[j]) return set_error(TNG_EINVAL, "unipc_step: orders (%d, %d) need history slot %d", p, q, j + 1);
    if (hist[j] == m_cur) return set_error(TNG_EINVAL, "unipc_step: m_cur aliases history slot %d", j + 1);
  }
  if (p > 0 && !last) return set_error(TNG_EINVAL, "unipc_step: corrector order %d needs last", p);
  const LatentStep ps{model_out, ld_mo, cfg, guidance, coef, prev, static_cast<__nv_bfloat16*>(next_in), ld_in,
                      split_off};
  return launch_latent_step("unipc_step", model_out && sample && m_cur, ps, B, C, HW,
                            UniPcStep{sample, p, q, m_cur, m_prev1, m_prev2, m_prev3, last}, stream);
}

extern "C" int tng_latent_blend(const float* x0, const float* noise, const float* mask, int64_t mask_bstride,
                                const float* coef, float* sample, void* next_in, int64_t ld_in, int32_t cfg,
                                int32_t split_off, int64_t B, int64_t C, int64_t HW, void* stream) {
  if (mask_bstride < 0) return set_error(TNG_EINVAL, "latent_blend: negative mask batch stride");
  const LatentStep p{nullptr, 0, cfg, 0.f, coef, sample, static_cast<__nv_bfloat16*>(next_in), ld_in, split_off};
  return launch_latent_step("latent_blend", x0 && sample, p, B, C, HW,
                            LatentBlend{x0, noise, mask, mask_bstride, sample}, stream);
}
