// camera.cuh -- the camera ray of a pixel (SH/RayGen.slang:35-50) and the tile partition's row map, shared by the path tracer's ray
// generation (wavefront_kernels.cu: camera_path) and the denoiser's feature pass (denoise_kernels.cu: k_features).
#pragma once
#include "shading.cuh"

namespace b200pt {

// partition helper (rank r owns rows y with ((y / band) % world) == r)
__host__ __device__ inline uint32_t part_global_row(uint32_t local_row, uint32_t rank, uint32_t world, uint32_t band) {
    uint32_t blk = local_row / band, in = local_row % band;
    return (blk * world + rank) * band + in;
}

// camera position before the depth-of-field offset (SH/RayGen.slang:41): the origin of every camera ray when DepthOfFieldStrength == 0
__device__ __forceinline__ float3 camera_eye(const DevConfig &cfg) {
    const float *VI = cfg.VI;
    return f3(VI[0] * 0.0f + VI[4] * 0.0f + VI[8] * 0.0f + VI[12] * 1.0f,
              VI[1] * 0.0f + VI[5] * 0.0f + VI[9] * 0.0f + VI[13] * 1.0f,
              VI[2] * 0.0f + VI[6] * 0.0f + VI[10] * 0.0f + VI[14] * 1.0f);
}

// Camera ray through pixel (x, y), SH/RayGen.slang:35-50.  Draws jitter x, jitter y, then the two lens samples (RandomCircleVec,
// SH/Sampler.slang:103-112) from rng.
__device__ __forceinline__ void camera_ray(const DevConfig &cfg, uint32_t x, uint32_t y, Rng &rng, float3 &ray_o, float3 &ray_d) {
    const float jx = rng.next() * (0.5f - -0.5f) + -0.5f;
    const float jy = rng.next() * (0.5f - -0.5f) + -0.5f;
    const float pcx = (float)x + 0.5f + jx, pcy = (float)y + 0.5f + jy;
    const float dx = (pcx / (float)cfg.W) * 2.0f - 1.0f, dy = (pcy / (float)cfg.H) * 2.0f - 1.0f;
    const float *VI = cfg.VI, *PI = cfg.PI;
    float3 origin = camera_eye(cfg);
    float3 target = f3(PI[0] * dx + PI[4] * dy + PI[8] * 1.0f + PI[12] * 1.0f,
                       PI[1] * dx + PI[5] * dy + PI[9] * 1.0f + PI[13] * 1.0f,
                       PI[2] * dx + PI[6] * dy + PI[10] * 1.0f + PI[14] * 1.0f);
    float3 direction = mat4_dir(VI, normalize(target));
    const float3 focus = origin + direction * fmaxf(cfg.FocusDistance, 0.001f);
    const float u1 = rng.next(), u2 = rng.next();
    const float theta = 2.0f * PT_PI * u1, rad = sqrtf(u2);
    const float ox = (rad * cosf(theta)) * 0.5f * cfg.DepthOfFieldStrength, oy = (rad * sinf(theta)) * 0.5f * cfg.DepthOfFieldStrength;
    origin = origin + (f3(VI[0], VI[1], VI[2]) * ox + f3(VI[4], VI[5], VI[6]) * oy);
    direction = normalize(focus - origin);
    ray_o = origin; ray_d = direction;
}

} // namespace b200pt
