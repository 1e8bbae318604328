// pose_kernels.cu -- glTF skinning and morph targets on the GPU (DESIGN §15).  Every pose is computed from the rest data uploaded at
// set_scene, never from the previous pose, so it depends only on (file, animation, t).
//   k_pose_vertices   one thread per vertex of the deformable meshes: morph deltas (targets of weight 0 skipped), the skin matrix blended
//                     over all influences, position M p, normal cof(M) n normalised as the loader normalises, uv plus its deltas
//   k_pose_normals    meshes loaded without NORMAL: each vertex's normal from the posed positions of the last face that uses it (the loader's
//                     "last face wins" rule, precomputed per vertex), so no scatter and no order dependence
// The loader's normalisation and face normals are restated with round-to-nearest intrinsics (no contraction into FMA), so an unskinned mesh
// at zero morph weights reproduces the vertices it was loaded with bit for bit.
#include "kernels.h"

namespace b200pt {

namespace {

__device__ __forceinline__ void normalize_like_loader(float &x, float &y, float &z) {   // n * (1 / sqrtf(|n|^2)), IEEE
    const float s = __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
    const float inv = __fdiv_rn(1.0f, __fsqrt_rn(s));
    x = __fmul_rn(x, inv); y = __fmul_rn(y, inv); z = __fmul_rn(z, inv);
}

__device__ __forceinline__ bool finite3(float a, float b, float c) { return isfinite(a) && isfinite(b) && isfinite(c); }

__global__ void __launch_bounds__(POSE_BLOCK) k_pose_vertices(const PoseDev d, bool smem_palette, b200pt_vertex *__restrict__ out, uint32_t *__restrict__ flag) {
    extern __shared__ float s_pal[];
    const PoseMesh D = d.meshes[d.block_mesh[blockIdx.x]];
    const float *pal = d.palette + (size_t)D.palette_base * 12;
    if ((D.flags & POSE_SKINNED) && smem_palette && D.n_joints <= POSE_SMEM_JOINTS) {
        for (uint32_t k = threadIdx.x; k < D.n_joints * 12; k += blockDim.x) s_pal[k] = pal[k];
        __syncthreads();
        pal = s_pal;
    }
    const uint32_t i = (blockIdx.x - D.block0) * blockDim.x + threadIdx.x;
    if (i >= D.count) return;
    const size_t v = (size_t)D.vbase + i;
    const float4 r0 = reinterpret_cast<const float4 *>(d.rest)[v * 2], r1 = reinterpret_cast<const float4 *>(d.rest)[v * 2 + 1];
    float p[3] = { r0.x, r0.y, r0.z }, n[3] = { r0.w, r1.x, r1.y }, uv[2] = { r1.z, r1.w };
    for (uint32_t t = 0; t < D.targets; t++) {
        const float w = d.morph[D.morph_base + t];
        if (w == 0.0f) continue;
        const float *pl = d.deltas + D.delta_base + (size_t)t * 8 * D.count + i;
        if (D.flags & POSE_DPOS) for (int c = 0; c < 3; c++) p[c] += w * __ldg(pl + (size_t)c * D.count);
        if (D.flags & POSE_DNRM) for (int c = 0; c < 3; c++) n[c] += w * __ldg(pl + (size_t)(3 + c) * D.count);
        if (D.flags & POSE_DUV) for (int c = 0; c < 2; c++) uv[c] += w * __ldg(pl + (size_t)(6 + c) * D.count);
    }
    if (D.flags & POSE_SKINNED) {
        float m[12];
        #pragma unroll
        for (int k = 0; k < 12; k++) m[k] = 0.0f;
        const uint4 *jj = reinterpret_cast<const uint4 *>(d.joints + D.jw_base + (size_t)i * 4 * D.sets);
        const float4 *ww = reinterpret_cast<const float4 *>(d.weights + D.jw_base + (size_t)i * 4 * D.sets);
        for (uint32_t s = 0; s < D.sets; s++) {
            const uint4 j = jj[s]; const float4 w = ww[s];
            const uint32_t js[4] = { j.x, j.y, j.z, j.w }; const float wsv[4] = { w.x, w.y, w.z, w.w };
            #pragma unroll
            for (int k = 0; k < 4; k++) {
                if (wsv[k] == 0.0f) continue;
                const float *J = pal + (size_t)js[k] * 12;
                #pragma unroll
                for (int e = 0; e < 12; e++) m[e] += wsv[k] * J[e];
            }
        }
        const float q[3] = { p[0], p[1], p[2] };
        for (int r = 0; r < 3; r++) p[r] = m[r * 4 + 0] * q[0] + m[r * 4 + 1] * q[1] + m[r * 4 + 2] * q[2] + m[r * 4 + 3];
        // cofactor of the upper 3x3: the inverse transpose times det(M), which the normalisation removes
        const float a = m[0], b = m[1], c = m[2], dd = m[4], e = m[5], f = m[6], g = m[8], h = m[9], k = m[10];
        const float c00 = e * k - f * h, c01 = f * g - dd * k, c02 = dd * h - e * g;
        const float c10 = h * c - k * b, c11 = k * a - g * c, c12 = g * b - h * a;
        const float c20 = b * f - c * e, c21 = c * dd - a * f, c22 = a * e - b * dd;
        const float nn[3] = { n[0], n[1], n[2] };
        n[0] = c00 * nn[0] + c01 * nn[1] + c02 * nn[2];
        n[1] = c10 * nn[0] + c11 * nn[1] + c12 * nn[2];
        n[2] = c20 * nn[0] + c21 * nn[1] + c22 * nn[2];
    }
    const bool gen = D.flags & POSE_GEN_NORMALS;
    if (gen) n[0] = n[1] = n[2] = 0.0f;                 // k_pose_normals writes them
    else normalize_like_loader(n[0], n[1], n[2]);
    b200pt_vertex o;
    o.Position[0] = p[0]; o.Position[1] = p[1]; o.Position[2] = p[2];
    o.Normal[0] = n[0]; o.Normal[1] = n[1]; o.Normal[2] = n[2];
    o.TexCoord[0] = uv[0]; o.TexCoord[1] = uv[1];
    float4 *dst = reinterpret_cast<float4 *>(out + v);
    dst[0] = make_float4(o.Position[0], o.Position[1], o.Position[2], o.Normal[0]);
    dst[1] = make_float4(o.Normal[1], o.Normal[2], o.TexCoord[0], o.TexCoord[1]);
    if (!finite3(p[0], p[1], p[2]) || !isfinite(uv[0]) || !isfinite(uv[1]) || (!gen && !finite3(n[0], n[1], n[2]))) atomicOr(flag, 1u);
}

__global__ void __launch_bounds__(POSE_BLOCK) k_pose_normals(const PoseDev d, b200pt_vertex *__restrict__ out, uint32_t *__restrict__ flag) {
    const PoseMesh D = d.meshes[d.block_mesh[blockIdx.x]];
    if (!(D.flags & POSE_GEN_NORMALS)) return;
    const uint32_t i = (blockIdx.x - D.block0) * blockDim.x + threadIdx.x;
    if (i >= D.count) return;
    const size_t v = (size_t)D.vbase + i;
    const uint32_t f = d.last_face[v];
    float nx = 0.0f, ny = 0.0f, nz = 0.0f;              // a vertex no face uses: (0, 0, 0), which the normalisation turns into NaN, as at load
    if (f != UINT32_MAX) {
        const uint32_t *tri = d.indices + D.ibase + (size_t)f * 3;
        const b200pt_vertex *base = out + D.vbase;
        const float *A = base[tri[0]].Position, *B = base[tri[1]].Position, *C = base[tri[2]].Position;
        const float e1[3] = { __fsub_rn(B[0], A[0]), __fsub_rn(B[1], A[1]), __fsub_rn(B[2], A[2]) };
        const float e2[3] = { __fsub_rn(C[0], A[0]), __fsub_rn(C[1], A[1]), __fsub_rn(C[2], A[2]) };
        nx = __fsub_rn(__fmul_rn(e1[1], e2[2]), __fmul_rn(e1[2], e2[1]));
        ny = __fsub_rn(__fmul_rn(e1[2], e2[0]), __fmul_rn(e1[0], e2[2]));
        nz = __fsub_rn(__fmul_rn(e1[0], e2[1]), __fmul_rn(e1[1], e2[0]));
        const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
        if (len > 0.0f) { nx = __fdiv_rn(nx, len); ny = __fdiv_rn(ny, len); nz = __fdiv_rn(nz, len); }
    }
    normalize_like_loader(nx, ny, nz);
    out[v].Normal[0] = nx; out[v].Normal[1] = ny; out[v].Normal[2] = nz;
    if (f != UINT32_MAX && !finite3(nx, ny, nz)) atomicOr(flag, 1u);
}

} // namespace

int launch_pose(const PoseDev &d, uint32_t n_blocks, uint32_t max_joints, bool gen_normals, b200pt_vertex *out, uint32_t *flag, cudaStream_t st) {
    if (!n_blocks) return 0;
    const uint32_t smem_joints = max_joints <= POSE_SMEM_JOINTS ? max_joints : 0;
    const size_t smem = (size_t)smem_joints * 12 * sizeof(float);
    k_pose_vertices<<<n_blocks, POSE_BLOCK, smem, st>>>(d, smem_joints > 0, out, flag);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    if (gen_normals) {
        k_pose_normals<<<n_blocks, POSE_BLOCK, 0, st>>>(d, out, flag);
        e = cudaGetLastError();
    }
    return (int)e;
}

} // namespace b200pt
