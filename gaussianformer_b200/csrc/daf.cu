// Deformable multi-camera / multi-scale aggregation (replaces deformable_aggregation_kernel and
// deformable_aggregation_grad_kernel, model/encoder/gaussian_encoder/ops/src/deformable_aggregation_cuda.cu:125-259).
//
// The reference runs one thread per output scalar: every thread re-reads the sampling location, the
// level table and its weight, and the backward issues one scalar atomic per corner, per weight and
// per location from every channel thread.  Here one WARP owns one sampling point:
//   * lanes span the channel vector in float4 slices, so each of the 4 bilinear corners is one
//     coalesced 16-byte-per-lane read of a 512-byte feature row (channels-last layout; 8 bytes per lane of a
//     256-byte row when the table is fp16 or bf16, converted to fp32 in registers);
//   * the camera gate and all bilinear coefficients are warp-uniform;
//   * backward: vector atomics for the feature gradients and shuffle reductions for the weight and
//     location gradients (visit_pairs, daf_pair.cuh) — no scalar atomic storms.
#include "daf_pair.cuh"
#include "gf_b200_debug.h"

namespace gf {

// Any C and Gr: a lane owns one channel per slice of 32 (shapes daf_fast_kernel does not take).
template <bool BACKWARD, class T>
__global__ void __launch_bounds__(kDafThreads) daf_kernel(const DafParams p) {
    const T *feat = static_cast<const T *>(p.feat);
    const int lane = threadIdx.x & 31;
    const int C = p.d.num_embeds, M = p.d.num_cams, L = p.d.num_scale, Gr = p.d.num_groups, F = p.d.num_feat;
    const int gdim = C / Gr;
    const long long npts = static_cast<long long>(p.d.batch) * p.d.num_pts;
    const long long warps = static_cast<long long>(gridDim.x) * (kDafThreads / 32);
    __shared__ int lh[kMaxLevels], lw[kMaxLevels], ls[kMaxLevels];
    load_level_table(p.d, p.shape, p.start, lh, lw, ls);

    for (long long bp = static_cast<long long>(blockIdx.x) * (kDafThreads / 32) + (threadIdx.x >> 5); bp < npts; bp += warps) {
        const int b = static_cast<int>(bp / p.d.num_pts);
        for (int c0 = lane; c0 < C; c0 += 32) {
            const int grp = c0 / gdim;
            float acc = 0.f;
            float gout = 0.f;
            if (BACKWARD) gout = __ldg(p.grad_out + bp * C + c0);
            for (int m = 0; m < M; ++m) {
                float lx, ly;
                if (!cam_gate(p.loc, bp, M, m, lx, ly)) continue;  // warp-uniform
                const T *fcam = feat + (static_cast<long long>(b) * M + m) * F * C + c0;
                const long long wbase = (bp * M + m) * static_cast<long long>(L) * Gr + grp;
                float gx = 0.f, gy = 0.f;
#pragma unroll 4
                for (int l = 0; l < L; ++l) {
                    const BilinearCell cell = bilinear_cell(lx, ly, lh[l], lw[l]);
                    const long long row0 = static_cast<long long>(cell.y0) * lw[l] + cell.x0;   // unclamped corner rows
                    const long long row[4] = {row0, row0 + 1, row0 + lw[l], row0 + lw[l] + 1};
                    const T *flev = fcam + static_cast<long long>(ls[l]) * C;
                    float v[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) v[k] = cell.inside(k, lh[l], lw[l]) ? load1(flev + row[k] * C) : 0.f;
                    const float wt = __ldg(p.weights + wbase + static_cast<long long>(l) * Gr);
                    // d(out)/d(x_im), d(out)/d(y_im)   (cuda.cu:85-121)
                    float dvx, dvy;
                    const float val = bilinear_value(cell, v, dvx, dvy);
                    if (!BACKWARD) {
                        acc = fmaf(wt, val, acc);
                    } else {
                        // d(out)/d(feat corner) = bilinear weight * aggregation weight
                        float *gf = p.grad_feat + (fcam - feat) + static_cast<long long>(ls[l]) * C;
#pragma unroll
                        for (int k = 0; k < 4; ++k)
                            if (cell.inside(k, lh[l], lw[l])) atomicAdd(gf + row[k] * C, (cell.weight(k) * wt) * gout);
                        // d(out)/d(weight) = sampled value
                        const float gw = gout * val;
                        gx = fmaf(static_cast<float>(lw[l]) * wt, gout * dvx, gx);
                        gy = fmaf(static_cast<float>(lh[l]) * wt, gout * dvy, gy);
                        atomicAdd(p.grad_weights + wbase + static_cast<long long>(l) * Gr, gw);
                    }
                }
                if (BACKWARD) {
                    float *gl = p.grad_loc + (bp * M + m) * 2;
                    atomicAdd(gl, gx);
                    atomicAdd(gl + 1, gy);
                }
            }
            if (!BACKWARD) p.out[bp * C + c0] = acc;
        }
    }
}

// The weight and location gradients of daf_kernel's shapes without floating-point atomics (the deterministic
// backward; its feature gradient is gathered in daf_det.cu).  One warp per point, a lane per group: the lane sums its
// group's channels in ascending order, so each weight gradient has one writer and a fixed order; the location
// gradient of a camera is the lanes' partial sums over the levels, reduced with a fixed shuffle tree.
template <class T>
__global__ void __launch_bounds__(kDafThreads) daf_det_generic_kernel(const DafParams p) {
    const T *feat = static_cast<const T *>(p.feat);
    const int lane = threadIdx.x & 31;
    const int C = p.d.num_embeds, M = p.d.num_cams, L = p.d.num_scale, Gr = p.d.num_groups, F = p.d.num_feat;
    const int gdim = C / Gr;
    const long long npts = static_cast<long long>(p.d.batch) * p.d.num_pts;
    const long long warps = static_cast<long long>(gridDim.x) * (kDafThreads / 32);
    __shared__ int lh[kMaxLevels], lw[kMaxLevels], ls[kMaxLevels];
    load_level_table(p.d, p.shape, p.start, lh, lw, ls);

    for (long long bp = static_cast<long long>(blockIdx.x) * (kDafThreads / 32) + (threadIdx.x >> 5); bp < npts; bp += warps) {
        const int b = static_cast<int>(bp / p.d.num_pts);
        const float *gop = p.grad_out + bp * C;
        for (int m = 0; m < M; ++m) {
            float lx, ly;
            if (!cam_gate(p.loc, bp, M, m, lx, ly)) continue;  // warp-uniform
            const T *fcam = feat + (static_cast<long long>(b) * M + m) * F * C;
            const long long wbase = (bp * M + m) * static_cast<long long>(L) * Gr;
            float gx = 0.f, gy = 0.f;
            for (int l = 0; l < L; ++l) {
                const BilinearCell cell = bilinear_cell(lx, ly, lh[l], lw[l]);
                const long long row0 = static_cast<long long>(cell.y0) * lw[l] + cell.x0;
                const long long row[4] = {row0, row0 + 1, row0 + lw[l], row0 + lw[l] + 1};
                const T *flev = fcam + static_cast<long long>(ls[l]) * C;
                for (int g = lane; g < Gr; g += 32) {
                    const float wt = __ldg(p.weights + wbase + static_cast<long long>(l) * Gr + g);
                    float gw = 0.f;
                    for (int c = g * gdim; c < (g + 1) * gdim; ++c) {
                        float v[4];
#pragma unroll
                        for (int k = 0; k < 4; ++k) v[k] = cell.inside(k, lh[l], lw[l]) ? load1(flev + row[k] * C + c) : 0.f;
                        const float gout = __ldg(gop + c);
                        float dvx, dvy;
                        const float val = bilinear_value(cell, v, dvx, dvy);
                        gw = fmaf(gout, val, gw);
                        gx = fmaf(static_cast<float>(lw[l]) * wt, gout * dvx, gx);
                        gy = fmaf(static_cast<float>(lh[l]) * wt, gout * dvy, gy);
                    }
                    p.grad_weights[wbase + static_cast<long long>(l) * Gr + g] += gw;
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                gx += __shfl_xor_sync(0xffffffffu, gx, o);
                gy += __shfl_xor_sync(0xffffffffu, gy, o);
            }
            if (lane == 0) {
                float *gl = p.grad_loc + (bp * M + m) * 2;
                gl[0] += gx;
                gl[1] += gy;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Fast path (C % 128 == 0, a group = whole lanes, M*L <= 32): one warp per sampling point, and the
// bilinear setup of each (camera, level) pair is computed by ONE lane instead of all 32 — a kernel
// that repeats it in every lane is instruction-bound (224 M warp instructions, L2 at 27 %), almost
// all of it redundant warp-uniform setup arithmetic.  The setup and the visit are setup_pairs and
// visit_pairs (daf_pair.cuh).
// ------------------------------------------------------------------------------------------------
template <bool BACKWARD, class T, bool FEAT_GRAD = true>
__global__ void __launch_bounds__(kDafThreads, BACKWARD ? 3 : 4) daf_fast_kernel(const DafParams p) {
    __shared__ int lh[kMaxLevels], lw[kMaxLevels], ls[kMaxLevels];
    __shared__ __align__(16) PairSetup s_pair[kDafThreads / 32][32];
    load_level_table(p.d, p.shape, p.start, lh, lw, ls);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int C = p.d.num_embeds, M = p.d.num_cams, L = p.d.num_scale, Gr = p.d.num_groups, F = p.d.num_feat;
    const int npair = M * L;
    const int gdim = C / Gr, lanes_per_group = gdim / 4;
    const long long npts = static_cast<long long>(p.d.batch) * p.d.num_pts;
    const long long warps = static_cast<long long>(gridDim.x) * (kDafThreads / 32);
    PairSetup *mine = s_pair[warp];
    const int my_cam = lane / L, my_lv = lane - my_cam * L;   // lane <-> (camera, level) pair, fixed for the kernel
    const bool small_index = npts < (1ll << 31);

    for (long long bp = static_cast<long long>(blockIdx.x) * (kDafThreads / 32) + warp; bp < npts; bp += warps) {
        const int b = small_index ? static_cast<int>(bp) / p.d.num_pts : static_cast<int>(bp / p.d.num_pts);
        const uint32_t visible = setup_pairs(p.d, p.loc, lh, lw, ls, bp, lane, my_cam, my_lv, nullptr, mine);
        const T *featb = static_cast<const T *>(p.feat) + static_cast<long long>(b) * M * F * C;
        float *gfeatb = p.grad_feat + static_cast<long long>(b) * M * F * C;
        const float *wpt = p.weights + bp * npair * Gr;
        for (int c0 = lane * 4; c0 < C; c0 += 128) {
            const int grp = c0 / gdim;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            float4 gout = make_float4(0.f, 0.f, 0.f, 0.f);
            if (BACKWARD) gout = __ldg(reinterpret_cast<const float4 *>(p.grad_out + bp * C + c0));
            visit_pairs<BACKWARD, FEAT_GRAD>(mine, visible, featb, gfeatb, c0, lane, lanes_per_group, gout, p.grad_loc, bp, M, acc,
                                  [=](int pr) { return __ldg(wpt + pr * Gr + grp); },
                                  [gwt = p.grad_weights, bp, npair, Gr, grp](int pr, float, float gw) { gwt[(bp * npair + pr) * Gr + grp] += gw; });
            if (!BACKWARD) *reinterpret_cast<float4 *>(p.out + bp * C + c0) = acc;
        }
        __syncwarp();   // the next point overwrites this warp's setup slots
    }
}

int launch_daf(const DafParams &p, int dtype, DafPass pass, int num_sms, cudaStream_t stream) {
    const long long npts = static_cast<long long>(p.d.batch) * p.d.num_pts;
    if (npts == 0) return GF_OK;
    const int grid = daf_grid(npts, num_sms);
    const bool v4 = daf_vec4_ok(p.d);
    return dispatch_feat_dtype(dtype, "daf", [&](auto tag) {
        using T = typename decltype(tag)::type;
        if (pass == DafPass::kForward) {
            if (v4) daf_fast_kernel<false, T><<<grid, kDafThreads, 0, stream>>>(p);
            else daf_kernel<false, T><<<grid, kDafThreads, 0, stream>>>(p);
        } else if (pass == DafPass::kBackward) {
            if (v4) daf_fast_kernel<true, T><<<grid, kDafThreads, 0, stream>>>(p);
            else daf_kernel<true, T><<<grid, kDafThreads, 0, stream>>>(p);
        } else {
            if (v4) daf_fast_kernel<true, T, false><<<grid, kDafThreads, 0, stream>>>(p);
            else daf_det_generic_kernel<T><<<grid, kDafThreads, 0, stream>>>(p);
        }
        GF_CUDA_TRY(cudaGetLastError());
        return GF_OK;
    });
}

// Random row gather: every warp sums rows of `row_floats` floats (a multiple of 128) picked by idx[] from a table -- the
// access pattern of the sampling op without its arithmetic.  A warp reads 32 row numbers with one coalesced load and
// keeps eight 512-byte row reads in flight (the op keeps four per visible pair).  With a table that fits L2 this
// measures the L2 -> SM gather bandwidth the op can reach at most.
__global__ void __launch_bounds__(256) gather_probe_kernel(const float *table, const int32_t *idx, long long n, int row_floats, float *sink) {
    const int lane = threadIdx.x & 31;
    const long long warp = (static_cast<long long>(blockIdx.x) * 256 + threadIdx.x) >> 5, warps = static_cast<long long>(gridDim.x) * 8;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long i = warp * 32; i < n; i += warps * 32) {
        const long long j = i + lane < n ? i + lane : n - 1;
        const int mine = __ldg(idx + j);
#pragma unroll 1
        for (int k0 = 0; k0 < 32; k0 += 8) {
            const float *row[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) row[k] = table + static_cast<long long>(__shfl_sync(0xffffffffu, mine, k0 + k)) * row_floats;
            for (int c0 = lane * 4; c0 < row_floats; c0 += 128) {
                float4 v[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) v[k] = __ldg(reinterpret_cast<const float4 *>(row[k] + c0));   // eight loads in flight
#pragma unroll
                for (int k = 0; k < 8; ++k) { acc.x += v[k].x; acc.y += v[k].y; acc.z += v[k].z; acc.w += v[k].w; }
            }
        }
    }
    if (acc.x + acc.y + acc.z + acc.w == 123456.789f) sink[0] = acc.x;   // keeps the loads alive
}

// ------------------------------------------------------------------------------------------------
// feature_maps_format: [B*M, C, hw_l] maps <-> channels-last table [B*M, F, C], one tiled transpose
// ------------------------------------------------------------------------------------------------
struct FormatParams {
    void *maps[GF_DAF_MAX_LEVELS];   // elements of the kernel's type T, like the table
    void *table;
    int hw[GF_DAF_MAX_LEVELS], start[GF_DAF_MAX_LEVELS], tile0[GF_DAF_MAX_LEVELS + 1];   // rows, first row, first tile of a level
    int L, C, F;
};

// Four consecutive elements of T, moved as one access: a float4 for float, 8 bytes for the 2-byte types.
template <class T>
struct __align__(8) Pack4 { T x, y, z, w; };
template <class T>
struct Vec4Of { using type = Pack4<T>; };
template <>
struct Vec4Of<float> { using type = float4; };

template <class T>
__device__ __forceinline__ typename Vec4Of<T>::type ldg_vec4(const T *p) {
    if constexpr (sizeof(T) == 4) {
        return __ldg(reinterpret_cast<const float4 *>(p));
    } else {
        const uint2 raw = __ldg(reinterpret_cast<const uint2 *>(p));
        return *reinterpret_cast<const Pack4<T> *>(&raw);
    }
}

// 64 (rows of the table) x 64 (channels) tiles through shared memory; both global sides move 4 elements
// (16 bytes for float, 8 for the 2-byte types) per thread along their contiguous axis (rows of a map,
// channels of the table).  Pure data movement in the maps' own type T.
template <bool INVERSE, class T>
__global__ void __launch_bounds__(256) daf_format_kernel(const FormatParams p) {
    using V = typename Vec4Of<T>::type;
    constexpr uintptr_t kVecMask = 4 * sizeof(T) - 1;
    __shared__ T tile[64][65];
    int lv = 0;
    while (lv + 1 < p.L && static_cast<int>(blockIdx.x) >= p.tile0[lv + 1]) ++lv;
    const int r0 = (blockIdx.x - p.tile0[lv]) * 64, c0 = blockIdx.y * 64;
    const int hw = p.hw[lv];
    const size_t bm = blockIdx.z;
    T *map = static_cast<T *>(p.maps[lv]) + bm * p.C * hw;                  // [C][hw]
    T *tab = static_cast<T *>(p.table) + (bm * p.F + p.start[lv]) * p.C;    // [hw][C]
    const int t = threadIdx.x;
    const bool vec_rows = (hw & 3) == 0 && (reinterpret_cast<uintptr_t>(map) & kVecMask) == 0;
    const bool vec_ch = (p.C & 3) == 0 && (reinterpret_cast<uintptr_t>(tab) & kVecMask) == 0;
    if (!INVERSE) {
        // map -> tile[row][channel]
        for (int i = t; i < 64 * 16; i += 256) {
            const int c = i >> 4, r4 = (i & 15) * 4;
            if (c0 + c >= p.C) continue;
            const T *src = map + static_cast<size_t>(c0 + c) * hw + r0 + r4;
            if (vec_rows && r0 + r4 + 3 < hw) {
                const V v = ldg_vec4(src);
                tile[r4][c] = v.x; tile[r4 + 1][c] = v.y; tile[r4 + 2][c] = v.z; tile[r4 + 3][c] = v.w;
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (r0 + r4 + k < hw) tile[r4 + k][c] = __ldg(src + k);
            }
        }
        __syncthreads();
        for (int i = t; i < 64 * 16; i += 256) {
            const int r = i >> 4, c4 = (i & 15) * 4;
            if (r0 + r >= hw || c0 + c4 >= p.C) continue;
            T *dst = tab + static_cast<size_t>(r0 + r) * p.C + c0 + c4;
            if (vec_ch && c0 + c4 + 3 < p.C) {
                *reinterpret_cast<V *>(dst) = V{tile[r][c4], tile[r][c4 + 1], tile[r][c4 + 2], tile[r][c4 + 3]};
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (c0 + c4 + k < p.C) dst[k] = tile[r][c4 + k];
            }
        }
    } else {
        // table -> tile[row][channel] -> map
        for (int i = t; i < 64 * 16; i += 256) {
            const int r = i >> 4, c4 = (i & 15) * 4;
            if (r0 + r >= hw || c0 + c4 >= p.C) continue;
            const T *src = tab + static_cast<size_t>(r0 + r) * p.C + c0 + c4;
            if (vec_ch && c0 + c4 + 3 < p.C) {
                const V v = ldg_vec4(src);
                tile[r][c4] = v.x; tile[r][c4 + 1] = v.y; tile[r][c4 + 2] = v.z; tile[r][c4 + 3] = v.w;
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (c0 + c4 + k < p.C) tile[r][c4 + k] = __ldg(src + k);
            }
        }
        __syncthreads();
        for (int i = t; i < 64 * 16; i += 256) {
            const int c = i >> 4, r4 = (i & 15) * 4;
            if (c0 + c >= p.C) continue;
            T *dst = map + static_cast<size_t>(c0 + c) * hw + r0 + r4;
            if (vec_rows && r0 + r4 + 3 < hw) {
                *reinterpret_cast<V *>(dst) = V{tile[r4][c], tile[r4 + 1][c], tile[r4 + 2][c], tile[r4 + 3][c]};
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (r0 + r4 + k < hw) dst[k] = tile[r4 + k][c];
            }
        }
    }
}

int launch_daf_format(const gf_daf_format_desc &d, int dtype, void *const *maps, void *table, bool inverse, cudaStream_t stream) {
    FormatParams fp{};
    fp.L = d.num_scale;
    fp.C = d.num_embeds;
    fp.table = table;
    int rows = 0, tiles = 0;
    for (int l = 0; l < d.num_scale; ++l) {
        fp.maps[l] = maps[l];
        fp.hw[l] = d.hw[l];
        fp.start[l] = rows;
        fp.tile0[l] = tiles;
        rows += d.hw[l];
        tiles += (d.hw[l] + 63) / 64;
    }
    fp.tile0[d.num_scale] = tiles;
    fp.F = rows;
    if (tiles == 0 || d.batch_cams == 0 || d.num_embeds == 0) return GF_OK;
    const dim3 grid(tiles, (d.num_embeds + 63) / 64, d.batch_cams);
    GF_REQUIRE(grid.y <= 65535 && grid.z <= 65535, GF_ERR_UNSUPPORTED, "daf format: too many channels or cameras");
    return dispatch_feat_dtype(dtype, "daf format", [&](auto tag) {
        using T = typename decltype(tag)::type;
        if (inverse) daf_format_kernel<true, T><<<grid, 256, 0, stream>>>(fp);
        else daf_format_kernel<false, T><<<grid, 256, 0, stream>>>(fp);
        GF_CUDA_TRY(cudaGetLastError());
        return GF_OK;
    });
}

}  // namespace gf

extern "C" int gf_debug_gather_probe(const float *table, const int32_t *idx, int64_t n, int32_t row_floats, float *sink,
                                     gf_stream_t stream_) {
    GF_REQUIRE(table && idx && sink && n > 0 && row_floats > 0 && row_floats % 128 == 0, GF_ERR_INVALID_ARG, "gather probe: bad argument");
    int dev = 0, num_sms = 1;
    GF_CUDA_TRY(cudaGetDevice(&dev));
    GF_CUDA_TRY(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    gf::gather_probe_kernel<<<num_sms * 8, 256, 0, static_cast<cudaStream_t>(stream_)>>>(table, idx, n, row_floats, sink);
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}
