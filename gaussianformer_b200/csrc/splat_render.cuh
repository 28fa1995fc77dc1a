// Shared pieces of the render kernels: launch parameters and the exact per-point evaluation
// (used by the generic kernel for every point and by the tile kernels for the rare point that
// is not in canonical voxel order).
#pragma once
#include "common.cuh"

namespace gf {

struct RenderParams {
    gf_splat_desc d;
    const float *pts;
    const int32_t *points_int;
    gf_splat_outputs out;
    SplatWorkspace ws;
    int nby;         // bins along y
    int nzc;         // z chunks
    int nbx;         // bins along x (blockIdx.z = sample * nbx + bin x)
    int ce_rows;     // rows of out.ce_partials per sample (= render CTAs per sample)
    int vec_ok;      // D % 4 == 0 and every tensor the tile kernel touches with 16-byte vectors is 16-byte aligned
};

// The launch parameters narrowed to sample b of the batch: per-sample input tensors and workspace blocks.  The output
// pointers are narrowed separately (with_sample_outputs) where they are needed, i.e. after the accumulation loop,
// so that they do not occupy registers during it.
__device__ __forceinline__ RenderParams with_sample_outputs(const RenderParams &p, const RenderParams &launch, int b) {
    RenderParams q = p;
    q.out = sample_outputs(launch.d, launch.out, b, launch.ce_rows);
    return q;
}
__device__ __forceinline__ RenderParams sample_params(const RenderParams &p, int b) {
    RenderParams q = p;
    gf_splat_inputs in = {};
    in.pts = p.pts;
    in.points_int = p.points_int;
    in = sample_inputs(p.d, in, b);
    q.pts = in.pts;
    q.points_int = in.points_int;
    q.ws = sample_ws(p.ws, p.d.G, b);
    return q;
}

// index of the largest of C values, lowest index on ties
template <int C>
__device__ __forceinline__ int argmax_of(const float (&v)[C]) {
    int best = 0;
    float bv = v[0];
#pragma unroll
    for (int c = 1; c < C; ++c)
        if (v[c] > bv) { bv = v[c]; best = c; }
    return best;
}

// Evaluate point n = (x,y,z) against the ascending Gaussian list of its supertile with the exact
// integer-box test and write its output row(s).  Follows FORWARD::renderCUDA
// (model/head/localagg/src/forward.cu:46-82; prob: localagg_prob/src/forward.cu:56-101).
template <int C, bool PROB>
__device__ __forceinline__ void render_one_point(const RenderParams &p, long long n, float x, float y, float z) {
    constexpr int REC = rec_floats(C);
    const int H = p.d.H, W = p.d.W, D = p.d.D;
    int ix, iy, iz;
    if (p.points_int) {
        ix = p.points_int[3 * n]; iy = p.points_int[3 * n + 1]; iz = p.points_int[3 * n + 2];
    } else {
        ix = voxel_coord(x, p.d.pc_min[0], p.d.grid_size);
        iy = voxel_coord(y, p.d.pc_min[1], p.d.grid_size);
        iz = voxel_coord(z, p.d.pc_min[2], p.d.grid_size);
    }
    float acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = 0.f;
    float zsum = 0.f, dens = 0.f, keep = 1.f;
    const bool ok = ix >= 0 && ix < H && iy >= 0 && iy < W && iz >= 0 && iz < D;
    if (!ok) {
        atomicOr(p.ws.flags, GF_FLAG_POINT_OUT_OF_GRID);
    } else {
        const int s = supertile_of(p.ws, ix, iy);
        const int ncand = p.ws.counts[s];
        const int32_t *cand = p.ws.lists + static_cast<size_t>(s) * p.d.G;
        for (int i = 0; i < ncand; ++i) {
            const int g = __ldg(cand + i);
            const uint4 b = __ldg(reinterpret_cast<const uint4 *>(p.ws.boxes) + g);
            const bool in = static_cast<uint32_t>(ix) >= (b.x & 0xffffu) && static_cast<uint32_t>(ix) <= (b.x >> 16) &&
                            static_cast<uint32_t>(iy) >= (b.y & 0xffffu) && static_cast<uint32_t>(iy) <= (b.y >> 16) &&
                            static_cast<uint32_t>(iz) >= (b.z & 0xffffu) && static_cast<uint32_t>(iz) <= (b.z >> 16) &&
                            b.w == 0u;
            if (!in) continue;
            const float4 *r4 = reinterpret_cast<const float4 *>(p.ws.records + static_cast<size_t>(g) * REC);
            const float4 g0 = __ldg(r4), g1 = __ldg(r4 + 1), g2 = __ldg(r4 + 2);
            const float dx = g0.x - x, dy = g0.y - y, dz = g0.z - z;
            float t1 = g1.x * dx;
            t1 = fmaf(g1.w, dy, t1);
            t1 = fmaf(g2.y, dz, t1);
            float t2 = g1.y * dy;
            t2 = fmaf(g2.x, dz, t2);
            float q = t1 * dx;
            q = fmaf(t2, dy, q);
            q = fmaf(g1.z * dz, dz, q);
            const float E = ex2_approx(q);
            const float w = PROB ? g0.w * E : E;   // base: the class vector of the record already carries the opacity
            if (PROB) {
                zsum += w;
                dens += E;
                keep *= (1.f - E);
            }
            // forward record layout (common.cuh): classes 0..15 in chunks 3..6, 16 17 in the coefficient chunk, 18 19 in chunk 7
#pragma unroll
            for (int c4 = 0; c4 < 4; ++c4) {
                const float4 s4 = __ldg(r4 + 3 + c4);
                const float sv[4] = {s4.x, s4.y, s4.z, s4.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) acc[c4 * 4 + k] = fmaf(sv[k], w, acc[c4 * 4 + k]);
            }
            if constexpr (C > 16) acc[16] = fmaf(g2.z, w, acc[16]);
            if constexpr (C > 17) acc[17] = fmaf(g2.w, w, acc[17]);
            if constexpr (C > 18) {
                const float4 s4 = __ldg(r4 + 7);
                acc[18] = fmaf(s4.x, w, acc[18]);
                if constexpr (C > 19) acc[19] = fmaf(s4.y, w, acc[19]);
            }
        }
    }
    if (PROB) {
        if (zsum > 1e-9f) {
#pragma unroll
            for (int c = 0; c < C; ++c) acc[c] = __fdiv_rn(acc[c], zsum);
        } else {
#pragma unroll
            for (int c = 0; c < C; ++c) acc[c] = (c < C - 1) ? static_cast<float>(1.0 / (C - 1)) : 0.f;
        }
        p.out.bin_logits[n] = 1.f - keep;
        p.out.density[n] = dens;
        p.out.probability[n] = zsum;
    }
#pragma unroll
    for (int c = 0; c < C; ++c) {
        if (p.out.logits) p.out.logits[n * C + c] = acc[c];
        if (p.out.logits_cn) p.out.logits_cn[static_cast<long long>(c) * p.d.N + n] = acc[c];
    }
    if (p.out.argmax) p.out.argmax[n] = static_cast<uint8_t>(argmax_of<C>(acc));
}

}  // namespace gf
