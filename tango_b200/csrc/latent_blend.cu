// latent_blend.cu — the latent-space blend of text-guided editing and inpainting, plus packing of the next UNet input,
// in one HBM pass. With a device coefficient row (sqrt_a, sqrt_1ma) it evaluates the schedulers' add_noise
// (scheduling_ddpm.py:351-372) and, under a mask, the legacy-inpaint blend (pipeline_stable_diffusion_inpaint_legacy.py:
// 692-709). Every product and sum is one IEEE round-to-nearest op in the fork's association order, so the result equals
// its fp32 CPU arithmetic bit for bit.
#include "tng_ptx.cuh"
#include "tng_internal.h"

namespace tng {

// One thread per latent element, walked in NCHW order (coalesced x0 / noise / sample / mask reads); the channels-last
// bf16 writes of a warp share their lines with the warps of the neighbouring channels, as in dpm_step_kernel.
__global__ void __launch_bounds__(256) latent_blend_kernel(const float* x0, const float* noise, const float* mask,
                                                            long long mask_bstride, const float* coef, float* sample,
                                                            __nv_bfloat16* next_in, long long ld_in, int cfg,
                                                            int split_off, long long B, int C, long long HW) {
  const float sqrt_a = coef[0], sqrt_1ma = coef[1];
  const long long total = B * C * HW;
  for (long long nchw = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; nchw < total;
       nchw += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long hw = nchw % HW;
    const int c = static_cast<int>((nchw / HW) % C);
    const long long b = nchw / (HW * C);
    // add_noise: sqrt_alpha_prod * original_samples + sqrt_one_minus_alpha_prod * noise
    float out = __fmul_rn(sqrt_a, x0[nchw]);
    if (noise) out = __fadd_rn(out, __fmul_rn(sqrt_1ma, noise[nchw]));
    if (mask) {
      // (init_latents_proper * mask) + (latents * (1 - mask))
      const float m = mask[b * mask_bstride + hw];
      out = __fadd_rn(__fmul_rn(out, m), __fmul_rn(sample[nchw], __fsub_rn(1.0f, m)));
    }
    sample[nchw] = out;
    if (next_in) {
      store_bf16_split(next_in + (b * HW + hw) * ld_in + c, out, split_off);
      if (cfg) store_bf16_split(next_in + ((B + b) * HW + hw) * ld_in + c, out, split_off);
    }
  }
}

}  // namespace tng

using namespace tng;

extern "C" int tng_latent_blend(const float* x0, const float* noise, const float* mask, int64_t mask_bstride,
                                const float* coef, float* sample, void* next_in, int64_t ld_in, int32_t cfg,
                                int32_t split_off, int64_t B, int64_t C, int64_t HW, void* stream) {
  if (!x0 || !coef || !sample) return set_error(TNG_EINVAL, "latent_blend: null argument");
  if (mask_bstride < 0) return set_error(TNG_EINVAL, "latent_blend: negative mask batch stride");
  if (next_in && ld_in < C + (split_off > 0 ? split_off : 0))
    return set_error(TNG_EINVAL, "latent_blend: ld_in %lld too small for %lld channels", (long long)ld_in, (long long)C);
  const long long total = B * C * HW;
  if (total < 1) return set_error(TNG_EINVAL, "latent_blend: empty shape");
  long long grid = (total + 255) / 256;
  const long long cap = 16LL * num_sms();   // grid-stride beyond 16 CTAs per SM
  if (grid > cap) grid = cap;
  latent_blend_kernel<<<static_cast<unsigned>(grid), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x0, noise, mask, mask_bstride, coef, sample, reinterpret_cast<__nv_bfloat16*>(next_in), ld_in, cfg, split_off, B,
      static_cast<int>(C), HW);
  return check_launch("latent_blend");
}
