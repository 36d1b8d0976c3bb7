// softras_launch.cuh -- launchers implemented in separate translation units (forward, backward) so that the template
// instantiations compile in parallel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

// pooled: optional [B,4,is/2,is/2] 2x2 mean of soft_colors written by the forward (anti-aliasing epilogue), or nullptr
cudaError_t b200r_launch_forward(const SoftRasParams& P, const SoftRasWorkspace& W, const float* textures, float* soft_colors,
                                 float* aggrs_info, int32_t* ids, float* pooled, int persistent, int exact, cudaStream_t st);
cudaError_t b200r_launch_backward(const SoftRasParams& P, const SoftRasWorkspace& W, const float* textures,
                                  const float* soft_colors, const float* aggrs_info, const int32_t* ids,
                                  const float* grad_soft_colors, float* grad_faces, float* grad_textures,
                                  int exact, cudaStream_t st);

// runs the statement(s) with D = P.dist_func and R = P.rgb_func as compile-time constants
#define B200R_DISPATCH_DIST_RGB(...)                                       \
    switch (P.dist_func * 3 + P.rgb_func) {                                \
        case 0: { constexpr int D = 0, R = 0; __VA_ARGS__; } break;        \
        case 1: { constexpr int D = 0, R = 1; __VA_ARGS__; } break;        \
        case 2: { constexpr int D = 0, R = 2; __VA_ARGS__; } break;        \
        case 3: { constexpr int D = 1, R = 0; __VA_ARGS__; } break;        \
        case 4: { constexpr int D = 1, R = 1; __VA_ARGS__; } break;        \
        case 5: { constexpr int D = 1, R = 2; __VA_ARGS__; } break;        \
        case 6: { constexpr int D = 2, R = 0; __VA_ARGS__; } break;        \
        case 7: { constexpr int D = 2, R = 1; __VA_ARGS__; } break;        \
        default: { constexpr int D = 2, R = 2; __VA_ARGS__; } break;       \
    }
