// dpm_solver.cu — fused CFG combine + multistep DPM-Solver / DPM-Solver++ update (order 1, 2 or 3) + packing of the
// next UNet input, in one HBM pass. The per-step scalars come from a host-computed coefficient row (see
// tango_b200/schedulers.py:DPMSolverMultistepScheduler); every product and sum below is one IEEE round-to-nearest op
// in the reference's association order, so the result equals the reference's fp32 CPU arithmetic bit for bit.
#include "tng_ptx.cuh"
#include "tng_internal.h"

namespace tng {

// One thread per latent element, walked in NCHW order: the reads and writes of sample, the history slots and prev are
// coalesced across the warp; a warp's channels-last model-output reads and bf16 input writes are 32 rows apart and
// share their lines with the warps of the neighbouring channels.
__global__ void __launch_bounds__(256) dpm_step_kernel(const float* mo, long long ld_mo, int cfg, float guidance,
                                                        const float* sample, const float* coef, int order, float* m0_out,
                                                        const float* m1_in, const float* m2_in, float* prev,
                                                        __nv_bfloat16* next_in, long long ld_in, int split_off,
                                                        long long B, int C, long long HW) {
  const float c_a = coef[0], c_b = coef[1], c_d = coef[2], c_s = coef[3], c_0 = coef[4], c_1 = coef[5], c_2 = coef[6];
  const float inv_r0 = coef[7], inv_r1 = coef[8], w_r = coef[9], inv_r01 = coef[10];
  const long long total = B * C * HW;
  for (long long nchw = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; nchw < total;
       nchw += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long hw = nchw % HW;
    const int c = static_cast<int>((nchw / HW) % C);
    const long long b = nchw / (HW * C);
    const float s = sample[nchw];
    float v;
    if (cfg) {
      const float u = mo[(b * HW + hw) * ld_mo + c];
      const float t = mo[((B + b) * HW + hw) * ld_mo + c];
      v = __fadd_rn(u, __fmul_rn(guidance, __fsub_rn(t, u)));  // models.py:246
    } else {
      v = mo[(b * HW + hw) * ld_mo + c];
    }
    // convert_model_output (scheduling_dpmsolver_multistep.py:243-281): all six (algorithm, prediction) pairs
    const float m0 = __fdiv_rn(__fadd_rn(__fmul_rn(c_a, s), __fmul_rn(c_b, v)), c_d);
    m0_out[nchw] = m0;
    // first-order update (:305-313); the higher orders add their D1 / D2 terms in the reference's order (:336-427)
    float x = __fsub_rn(__fmul_rn(c_s, s), __fmul_rn(c_0, m0));
    if (order == 2) {
      const float d1 = __fmul_rn(inv_r0, __fsub_rn(m0, m1_in[nchw]));
      x = __fadd_rn(x, __fmul_rn(c_1, d1));
    } else if (order == 3) {
      const float m1 = m1_in[nchw];
      const float d1_0 = __fmul_rn(inv_r0, __fsub_rn(m0, m1));
      const float d1_1 = __fmul_rn(inv_r1, __fsub_rn(m1, m2_in[nchw]));
      const float dd = __fsub_rn(d1_0, d1_1);
      const float d1 = __fadd_rn(d1_0, __fmul_rn(w_r, dd));
      const float d2 = __fmul_rn(inv_r01, dd);
      x = __fsub_rn(__fadd_rn(x, __fmul_rn(c_1, d1)), __fmul_rn(c_2, d2));
    }
    if (prev) prev[nchw] = x;
    if (next_in) {
      store_bf16_split(next_in + (b * HW + hw) * ld_in + c, x, split_off);
      if (cfg) store_bf16_split(next_in + ((B + b) * HW + hw) * ld_in + c, x, split_off);
    }
  }
}

}  // namespace tng

using namespace tng;

extern "C" int tng_dpm_step(const float* model_out, int64_t ld_mo, int32_t cfg, float guidance, const float* sample,
                            const float* coef, int32_t order, float* m0, const float* m1, const float* m2, float* prev,
                            void* next_in, int64_t ld_in, int32_t split_off, int64_t B, int64_t C, int64_t HW,
                            void* stream) {
  if (!model_out || !sample || !coef || !m0 || (!prev && !next_in)) return set_error(TNG_EINVAL, "dpm_step: null argument");
  if (order < 1 || order > 3) return set_error(TNG_EINVAL, "dpm_step: order %d is not 1, 2 or 3", order);
  if ((order >= 2 && !m1) || (order == 3 && !m2)) return set_error(TNG_EINVAL, "dpm_step: order %d needs its history", order);
  const long long total = B * C * HW;
  if (total < 1) return set_error(TNG_EINVAL, "dpm_step: empty shape");
  long long grid = (total + 255) / 256;
  const long long cap = 16LL * num_sms();   // grid-stride beyond 16 CTAs per SM
  if (grid > cap) grid = cap;
  dpm_step_kernel<<<static_cast<unsigned>(grid), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      model_out, ld_mo, cfg, guidance, sample, coef, order, m0, m1, m2, prev, reinterpret_cast<__nv_bfloat16*>(next_in),
      ld_in, split_off, B, static_cast<int>(C), HW);
  return check_launch("dpm_step");
}
