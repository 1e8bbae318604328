// post_kernels.cu -- bloom mip chain + ACES tonemap (sm_90a), HBM-streaming kernels.
// Restates PathTracer/Shaders/PostProcess/{BloomDownSample,BloomUpSample,Tonemap}.slang as dispatched by
// PathTracer/PostProcessor.cpp:193-246.  Images are float4 (RGBA32F) row-major; every thread handles one pixel with
// 16-B coalesced accesses; the 16 taps of the down/up filters hit L1/L2 (each source texel is read by 4 neighbours).
#include "shading.cuh"
#include "kernels.h"

namespace b200pt {

// Every arithmetic step that more than one kernel evaluates is written with explicit-rounding intrinsics (no FMA contraction) in the
// operation order of the oracle (oracle/post_oracle.c): the fused chain below and the pass-per-pass chain produce bit-identical
// images (tests/test_gpu_parity.py::test_fused_post_chain_equals_pass_per_pass).  Divisions and pow follow the build's precision class
// (2-ulp division and exp2(y * log2 x) by default -- the forms SPIR-V grants the reference's shaders; IEEE / libm with PRECISE=1):
// ncu showed the chain's last kernel compute-bound (208 us for 185 MB of traffic) on libm powf and IEEE division sequences.
__device__ __forceinline__ float post_pow(float x, float y) {
#ifdef B200PT_PRECISE
    return powf(x, y);
#else
    return x > 0.0f ? exp2f(__fmul_rn(y, __log2f(x))) : (x == 0.0f ? 0.0f : __int_as_float(0x7FC00000));   // pow(0, y>0) = 0, pow(x<0, non-integer) = NaN
#endif
}
__device__ __forceinline__ float smoothstepf(float e0, float e1, float x) {
    const float t = clampf(__fsub_rn(x, e0) / __fsub_rn(e1, e0), 0.0f, 1.0f);
    return __fmul_rn(__fmul_rn(t, t), __fsub_rn(3.0f, __fmul_rn(2.0f, t)));
}
// BloomDownSample.slang:32-45 (FirstDispatch): one thresholded texel
__device__ __forceinline__ float3 bloom_threshold_px(float4 s, float start, float end) {
    const float br = __fadd_rn(__fadd_rn(__fmul_rn(s.x, 0.2126f), __fmul_rn(s.y, 0.7152f)), __fmul_rn(s.z, 0.0722f));
    const float f = smoothstepf(start, end, br);
    return f3(__fmul_rn(s.x, f), __fmul_rn(s.y, f), __fmul_rn(s.z, f));
}
__device__ __forceinline__ float bloom_scale(float acc, float strength) { return __fmul_rn(acc / 25.0f, strength); }   // /25 (Q14), *strength
__device__ __forceinline__ float mix_rn(float p, float q, float w) { return __fadd_rn(p, __fmul_rn(w, __fsub_rn(q, p))); }

__global__ void __launch_bounds__(256) k_bloom_threshold(const float4 *__restrict__ hdr, float4 *__restrict__ mip0, uint32_t npix, PostParams p) {
    const float start = p.BloomThreshold - p.FalloffRange, end = p.BloomThreshold + p.FalloffRange;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += gridDim.x * blockDim.x) {
        const float3 t = bloom_threshold_px(hdr[i], start, end);
        mip0[i] = make_float4(t.x, t.y, t.z, 1.0f);
    }
}

// BloomDownSample.slang:46-64 : taps 2*xy + (a,b), a,b in [-2,1], clamp, /25, *strength (Q14).
// Every chain kernel works on a ROW RANGE [y0, y1) of its destination (the whole image by default): a multi-GPU post pass gives each rank a block
// of output rows plus the halo rows the later passes read (Engine::post_process_rows).
__global__ void __launch_bounds__(256) k_bloom_down(const float4 *__restrict__ src, int sw, int sh, float4 *__restrict__ dst, int dw, int dh, PostParams p, int y0, int y1) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = y0 + blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= dw || y >= y1) return;
    float3 acc = f3(0.0f);
    #pragma unroll
    for (int a = -2; a < 2; a++) {
        #pragma unroll
        for (int b = -2; b < 2; b++) {
            const int sx = clampi(x * 2 + a, 0, sw - 1), sy = clampi(y * 2 + b, 0, sh - 1);
            const float4 s = __ldg(src + (size_t)sy * sw + sx);
            acc.x = __fadd_rn(acc.x, s.x); acc.y = __fadd_rn(acc.y, s.y); acc.z = __fadd_rn(acc.z, s.z);
        }
    }
    dst[(size_t)y * dw + x] = make_float4(bloom_scale(acc.x, p.BloomStrength), bloom_scale(acc.y, p.BloomStrength), bloom_scale(acc.z, p.BloomStrength), 1.0f);
}
// Fused first two dispatches of the chain (threshold + down-sample into mip 1): mip 0 is never written.  A 32 x 8 block of mip-1 texels
// needs the 66 x 18 HDR texels around it; each is thresholded ONCE into shared memory (it feeds up to 4 outputs) and the 16 taps of an
// output are read from there in the reference's order.  Clamping happens on the load, so tile slot (lx, ly) always holds the texel the
// clamped tap coordinate 2*x0 - 2 + lx would fetch.
__global__ void __launch_bounds__(256) k_bloom_down_first(const float4 *__restrict__ hdr, int sw, int sh, float4 *__restrict__ dst, int dw, int dh, PostParams p, int row0, int row1) {
    __shared__ float tr[18][66], tg[18][66], tb[18][66];
    const int x0 = blockIdx.x * 32, y0 = row0 + blockIdx.y * 8;
    const float start = p.BloomThreshold - p.FalloffRange, end = p.BloomThreshold + p.FalloffRange;
    for (int k = threadIdx.x; k < 66 * 18; k += 256) {
        const int lx = k % 66, ly = k / 66;
        const int gx = clampi(2 * x0 - 2 + lx, 0, sw - 1), gy = clampi(2 * y0 - 2 + ly, 0, sh - 1);
        const float3 t = bloom_threshold_px(__ldg(hdr + (size_t)gy * sw + gx), start, end);
        tr[ly][lx] = t.x; tg[ly][lx] = t.y; tb[ly][lx] = t.z;
    }
    __syncthreads();
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int x = x0 + tx, y = y0 + ty;
    if (x >= dw || y >= row1) return;
    float3 acc = f3(0.0f);
    #pragma unroll
    for (int a = -2; a < 2; a++) {
        #pragma unroll
        for (int b = -2; b < 2; b++) {
            const int lx = 2 * tx + a + 2, ly = 2 * ty + b + 2;
            acc.x = __fadd_rn(acc.x, tr[ly][lx]); acc.y = __fadd_rn(acc.y, tg[ly][lx]); acc.z = __fadd_rn(acc.z, tb[ly][lx]);
        }
    }
    dst[(size_t)y * dw + x] = make_float4(bloom_scale(acc.x, p.BloomStrength), bloom_scale(acc.y, p.BloomStrength), bloom_scale(acc.z, p.BloomStrength), 1.0f);
}

// BloomUpSample.slang:21-48 : taps xy/2 + (a,b) + 1, clamp, /25, *strength
__device__ __forceinline__ float3 bloom_up_taps(const float4 *__restrict__ src, int sw, int sh, int x, int y, float strength) {
    float3 acc = f3(0.0f);
    #pragma unroll
    for (int a = -2; a < 2; a++) {
        #pragma unroll
        for (int b = -2; b < 2; b++) {
            const int sx = clampi(x / 2 + a + 1, 0, sw - 1), sy = clampi(y / 2 + b + 1, 0, sh - 1);
            const float4 s = __ldg(src + (size_t)sy * sw + sx);
            acc.x = __fadd_rn(acc.x, s.x); acc.y = __fadd_rn(acc.y, s.y); acc.z = __fadd_rn(acc.z, s.z);
        }
    }
    return f3(bloom_scale(acc.x, strength), bloom_scale(acc.y, strength), bloom_scale(acc.z, strength));
}
// ... added to the finer mip in place
__global__ void __launch_bounds__(256) k_bloom_up(const float4 *__restrict__ src, int sw, int sh, float4 *__restrict__ dst, int dw, int dh, PostParams p, int y0, int y1) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = y0 + blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= dw || y >= y1) return;
    const float3 u = bloom_up_taps(src, sw, sh, x, y, p.BloomStrength);
    const float4 cur = dst[(size_t)y * dw + x];
    dst[(size_t)y * dw + x] = make_float4(__fadd_rn(u.x, cur.x), __fadd_rn(u.y, cur.y), __fadd_rn(u.z, cur.z), 1.0f);
}

// Tonemap.slang:20-55
__device__ __forceinline__ float3 aces_fitted(float3 c) {
    float3 v = f3(0.59719f * c.x + 0.35458f * c.y + 0.04823f * c.z,
                  0.07600f * c.x + 0.90834f * c.y + 0.01566f * c.z,
                  0.02840f * c.x + 0.13383f * c.y + 0.83777f * c.z);
    float3 a = f3(v.x * (v.x + 0.0245786f) - 0.000090537f, v.y * (v.y + 0.0245786f) - 0.000090537f, v.z * (v.z + 0.0245786f) - 0.000090537f);
    float3 b = f3(v.x * (0.983729f * v.x + 0.4329510f) + 0.238081f, v.y * (0.983729f * v.y + 0.4329510f) + 0.238081f, v.z * (0.983729f * v.z + 0.4329510f) + 0.238081f);
    float3 r = a / b;
    return f3(clampf(1.60475f * r.x + -0.53108f * r.y + -0.07367f * r.z, 0.0f, 1.0f),
              clampf(-0.10208f * r.x + 1.10813f * r.y + -0.00605f * r.z, 0.0f, 1.0f),
              clampf(-0.00327f * r.x + -0.07276f * r.y + 1.07602f * r.z, 0.0f, 1.0f));
}
__device__ __forceinline__ unsigned char unorm8(float q) {
    if (!(q > 0.0f)) q = 0.0f;
    if (q > 1.0f) q = 1.0f;
    return (unsigned char)__float2int_rn(q * 255.0f);
}
// Tonemap.slang:159-175 after the bloom fetch: (HDR + bloom) * exposure -> pow(1/gamma) -> ACES -> RGBA8 (Q15).  One compiled copy
// (noinline) serves k_tonemap and k_bloom_final, so both round identically.
static __device__ __noinline__ uchar4 tonemap_px(float3 h, float3 bl, float exposure, float gamma) {
    float3 c = f3(__fmul_rn(__fadd_rn(h.x, bl.x), exposure), __fmul_rn(__fadd_rn(h.y, bl.y), exposure), __fmul_rn(__fadd_rn(h.z, bl.z), exposure));
    const float ig = 1.0f / gamma;
    c = f3(post_pow(c.x, ig), post_pow(c.y, ig), post_pow(c.z, ig));
    const float3 o = aces_fitted(c);
    return make_uchar4(unorm8(o.x), unorm8(o.y), unorm8(o.z), 255);
}
// bilinear footprint of the bloom fetch: uv = xy / size, CLAMP_TO_EDGE, texel centres at +0.5
struct BloomTap { int x0, x1, y0, y1; float ax, ay; };
__device__ __forceinline__ BloomTap bloom_tap(int x, int y, int W, int H) {
    const float u = (float)x / (float)W, v = (float)y / (float)H;
    const float fxp = __fsub_rn(__fmul_rn(u, (float)W), 0.5f), fyp = __fsub_rn(__fmul_rn(v, (float)H), 0.5f);
    const float fx = floorf(fxp), fy = floorf(fyp);
    BloomTap t;
    t.ax = __fsub_rn(fxp, fx); t.ay = __fsub_rn(fyp, fy);
    t.x0 = clampi((int)fx, 0, W - 1); t.x1 = clampi((int)fx + 1, 0, W - 1);
    t.y0 = clampi((int)fy, 0, H - 1); t.y1 = clampi((int)fy + 1, 0, H - 1);
    return t;
}
__device__ __forceinline__ float3 bloom_blend(float4 t00, float4 t10, float4 t01, float4 t11, float ax, float ay) {
    return f3(mix_rn(mix_rn(t00.x, t10.x, ax), mix_rn(t01.x, t11.x, ax), ay),
              mix_rn(mix_rn(t00.y, t10.y, ax), mix_rn(t01.y, t11.y, ax), ay),
              mix_rn(mix_rn(t00.z, t10.z, ax), mix_rn(t01.z, t11.z, ax), ay));
}
__global__ void __launch_bounds__(256) k_tonemap(const float4 *__restrict__ hdr, const float4 *__restrict__ bloom0, uchar4 *__restrict__ ldr, int W, int H, PostParams p) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= W || y >= H) return;
    const BloomTap t = bloom_tap(x, y, W, H);
    const float4 t00 = __ldg(bloom0 + (size_t)t.y0 * W + t.x0), t10 = __ldg(bloom0 + (size_t)t.y0 * W + t.x1);
    const float4 t01 = __ldg(bloom0 + (size_t)t.y1 * W + t.x0), t11 = __ldg(bloom0 + (size_t)t.y1 * W + t.x1);
    const float4 h4 = hdr[(size_t)y * W + x];
    ldr[(size_t)y * W + x] = tonemap_px(f3(h4), bloom_blend(t00, t10, t01, t11, t.ax, t.ay), p.Exposure, p.Gamma);
}

// Fused last stage of the chain: [up-sample mip 1 into mip 0] + [threshold of the HDR image = the mip-0 term it is added to] + [tonemap].
// The reference materialises mip 0 three times (threshold write, up-sample read-modify-write, tonemap read: 5 x 16 B per pixel); here
// a 33 x 9 tile of mip 0 (the 32 x 8 output pixels + the one-texel halo the bilinear bloom fetch reaches to the left / top) is built in
// shared memory from the HDR image and mip 1 and consumed on the spot: HBM sees the HDR read, the small mip-1 read and the RGBA8 write.
// mip0_out (optional) receives the tile interior so GetBloom-style consumers can still see mip 0.
__global__ void __launch_bounds__(256) k_bloom_final(const float4 *__restrict__ hdr, const float4 *__restrict__ mip1, int mw, int mh,
                                                     uchar4 *__restrict__ ldr, float4 *__restrict__ mip0_out, int W, int H, PostParams p, int row0, int row1) {
    __shared__ float4 tile[9][34];      // bloom mip 0 (rgb), halo at row / column 0
    __shared__ float4 tile_h[9][34];    // HDR texel of the same pixel
    __shared__ float4 up[5][18];        // the up-sampled term: it depends on (x/2, y/2) only, so the 33 x 9 pixels share <= 17 x 5 values
    const int tx0 = blockIdx.x * 32, ty0 = row0 + blockIdx.y * 8;
    const int mx0 = clampi(tx0 - 1, 0, W - 1) / 2, my0 = clampi(ty0 - 1, 0, H - 1) / 2;
    const float start = p.BloomThreshold - p.FalloffRange, end = p.BloomThreshold + p.FalloffRange;
    for (int k = threadIdx.x; k < 17 * 5; k += 256) {
        const int ux = k % 17, uy = k / 17;
        const float3 u = bloom_up_taps(mip1, mw, mh, 2 * (mx0 + ux), 2 * (my0 + uy), p.BloomStrength);   // taps of every pixel with x/2 == mx0+ux, y/2 == my0+uy
        up[uy][ux] = make_float4(u.x, u.y, u.z, 0.0f);
    }
    for (int k = threadIdx.x; k < 33 * 9; k += 256) {
        const int lx = k % 33, ly = k / 33;
        const int gx = clampi(tx0 - 1 + lx, 0, W - 1), gy = clampi(ty0 - 1 + ly, 0, H - 1);
        tile_h[ly][lx] = __ldg(hdr + (size_t)gy * W + gx);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < 33 * 9; k += 256) {
        const int lx = k % 33, ly = k / 33;
        const int gx = clampi(tx0 - 1 + lx, 0, W - 1), gy = clampi(ty0 - 1 + ly, 0, H - 1);
        const float3 cur = bloom_threshold_px(tile_h[ly][lx], start, end);  // mip 0 before the up pass
        const float4 u = up[gy / 2 - my0][gx / 2 - mx0];
        tile[ly][lx] = make_float4(__fadd_rn(u.x, cur.x), __fadd_rn(u.y, cur.y), __fadd_rn(u.z, cur.z), 1.0f);
    }
    __syncthreads();
    const int x = tx0 + (threadIdx.x & 31), y = ty0 + (threadIdx.x >> 5);
    if (x >= W || y >= row1) return;
    const BloomTap t = bloom_tap(x, y, W, H);                               // x0 in {x-1, x}, x1 = x0 + 1 (clamped): inside the tile + halo
    const int lx0 = t.x0 - (tx0 - 1), lx1 = t.x1 - (tx0 - 1), ly0 = t.y0 - (ty0 - 1), ly1 = t.y1 - (ty0 - 1);
    const int cx = (threadIdx.x & 31) + 1, cy = (threadIdx.x >> 5) + 1;
    ldr[(size_t)y * W + x] = tonemap_px(f3(tile_h[cy][cx]), bloom_blend(tile[ly0][lx0], tile[ly0][lx1], tile[ly1][lx0], tile[ly1][lx1], t.ax, t.ay), p.Exposure, p.Gamma);
    if (mip0_out) mip0_out[(size_t)y * W + x] = tile[cy][cx];
}

// SH/RayGen.slang:130-137 as a stand-alone pass: fold one frame's radiance image into the accumulation image with the running-mean rule
// lerp(prev, new, 1 / (FrameCount + 1)) -- the "HDR accumulate" stage of BASELINE config 5 (inside PathTrace the same rule runs in k_resolve).
__global__ void __launch_bounds__(256) k_accumulate(const float4 *__restrict__ frame, float4 *__restrict__ image, uint32_t first, uint32_t count, uint32_t frame_index) {
    const float a = 1.0f / (float)(frame_index + 1u);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        const float4 s4 = frame[first + i];
        float3 c = f3(s4);
        if (frame_index > 0u) c = mix3(f3(image[first + i]), c, a);
        image[first + i] = make_float4(c.x, c.y, c.z, 1.0f);
    }
}
void launch_accumulate(const float4 *frame, float4 *image, uint32_t first, uint32_t count, uint32_t frame_index, int grid, cudaStream_t st) {
    if (count) k_accumulate<<<grid, 256, 0, st>>>(frame, image, first, count, frame_index);
}

void launch_bloom_threshold(const float4 *hdr, float4 *mip0, uint32_t npix, PostParams p, int grid, cudaStream_t st) {
    k_bloom_threshold<<<grid, 256, 0, st>>>(hdr, mip0, npix, p);
}
// rows == nullptr: the whole destination; else rows[0] <= y < rows[1]
static inline void row_range(const int *rows, uint32_t h, int &y0, int &y1) { y0 = rows ? rows[0] : 0; y1 = rows ? rows[1] : (int)h; if (y0 < 0) y0 = 0; if (y1 > (int)h) y1 = (int)h; }
void launch_bloom_down(const float4 *src, uint32_t sw, uint32_t sh, float4 *dst, uint32_t dw, uint32_t dh, PostParams p, cudaStream_t st, const int *rows) {
    int y0, y1; row_range(rows, dh, y0, y1); if (y1 <= y0) return;
    dim3 g((dw + 31) / 32, (y1 - y0 + 7) / 8);
    k_bloom_down<<<g, 256, 0, st>>>(src, (int)sw, (int)sh, dst, (int)dw, (int)dh, p, y0, y1);
}
void launch_bloom_down_first(const float4 *hdr, uint32_t W, uint32_t H, float4 *mip1, uint32_t dw, uint32_t dh, PostParams p, cudaStream_t st, const int *rows) {
    int y0, y1; row_range(rows, dh, y0, y1); if (y1 <= y0) return;
    dim3 g((dw + 31) / 32, (y1 - y0 + 7) / 8);
    k_bloom_down_first<<<g, 256, 0, st>>>(hdr, (int)W, (int)H, mip1, (int)dw, (int)dh, p, y0, y1);
}
void launch_bloom_final(const float4 *hdr, const float4 *mip1, uint32_t mw, uint32_t mh, uchar4 *ldr, float4 *mip0_out, uint32_t W, uint32_t H, PostParams p, cudaStream_t st, const int *rows) {
    int y0, y1; row_range(rows, H, y0, y1); if (y1 <= y0) return;
    dim3 g((W + 31) / 32, (y1 - y0 + 7) / 8);
    k_bloom_final<<<g, 256, 0, st>>>(hdr, mip1, (int)mw, (int)mh, ldr, mip0_out, (int)W, (int)H, p, y0, y1);
}
void launch_bloom_up(const float4 *src, uint32_t sw, uint32_t sh, float4 *dst, uint32_t dw, uint32_t dh, PostParams p, cudaStream_t st, const int *rows) {
    int y0, y1; row_range(rows, dh, y0, y1); if (y1 <= y0) return;
    dim3 g((dw + 31) / 32, (y1 - y0 + 7) / 8);
    k_bloom_up<<<g, 256, 0, st>>>(src, (int)sw, (int)sh, dst, (int)dw, (int)dh, p, y0, y1);
}
void launch_tonemap(const float4 *hdr, const float4 *bloom0, uchar4 *ldr, uint32_t W, uint32_t H, PostParams p, cudaStream_t st) {
    dim3 g((W + 31) / 32, (H + 7) / 8);
    k_tonemap<<<g, 256, 0, st>>>(hdr, bloom0, ldr, (int)W, (int)H, p);
}

} // namespace b200pt
