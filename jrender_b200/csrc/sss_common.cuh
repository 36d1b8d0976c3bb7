// sss_common.cuh -- what the forward (sss_api.cu) and the gradients (sss_grad_api.cu) of the texture-space subsurface
// scattering share: the blur's constants, one pass's parameters, and the forward's two pass kernels, which the backward
// launches again to recompute the intermediates the forward drops.
#pragma once

namespace b200r_sss {

constexpr int kTaps = 7;              // tap_num, lighting.py:117
constexpr int kMaxLevels = 8;
constexpr int kBlockX = 32, kBlockY = 8;

struct SssPass {
    const float* s_in;      // stretch map of the previous level [H, W]
    float* s_out;           // this level's blurred stretch map, or NULL (last level: nobody reads it)
    const float* irr_in;    // [3, H, W]
    float* irr_out;         // [3, H, W], or NULL (last y pass)
    float* acc;             // y passes: [3, H, W] running weighted sum of the levels
    const float* irr0;      // last y pass: the unblurred irradiance map [3, H, W]
    const float* spec;      // last y pass: the specular map [3, H, W]
    float* out;             // last y pass: [H, W, 3], rows flipped
    float taps[kTaps];
    float width;            // GaussWidth = float32(sqrt(v))
    float weight[3];        // y passes: this level's weight per channel
    int H, W, first, last;
};

using PassKernel = void (*)(SssPass);
// k_sss_blur_x / k_sss_blur_y of sss_api.cu
void forward_kernels(PassKernel* x_pass, PassKernel* y_pass);

}  // namespace b200r_sss
