// Pieces shared by the deformable-aggregation kernels (daf.cu, daf_fused.cu, daf_det.cu): their launch parameters, the
// level table, the sampling arithmetic, and the one-warp-per-point visit of the fast kernels (daf_fast_kernel,
// daf_fused_kernel):
//   lane p < M*L      : pair p = (camera p / L, level p % L): gate, 4 corner rows (clamped to a valid row), 4 corner
//                       weights (zero for corners outside the map) -> per-warp smem          (setup_pairs)
//   ballot of the gate: only visible pairs are visited, in ascending (camera, level) order   (visit_pairs)
//   every visit       : 2-3 uniform LDS.128 for the setup, one weight, 4 coalesced row loads per lane (16 bytes
//                       each for a float table, 8 for a half one), 16 FMAs
//   backward          : 16-byte vector atomics for the feature gradient, the weight gradient reduced over the lanes
//                       of a group with shuffles and handed to one lane, the location gradient reduced over the warp
//                       once per visible camera
// The feature table is float, __half or __nv_bfloat16 (the kernels are templated on its element type T); every value
// is converted to fp32 where it is loaded, so the arithmetic and the feature gradient are fp32 for all three.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace gf {

constexpr int kDafThreads = 256;
constexpr int kMaxLevels = 8;

template <class T>
struct TypeTag { using type = T; };

// f(TypeTag<T>{}) for the element type T of a GF_DTYPE_* code; any other code is reported as `what`'s error.
template <class F>
int dispatch_feat_dtype(int dtype, const char *what, F &&f) {
    switch (dtype) {
    case GF_DTYPE_F32: return f(TypeTag<float>{});
    case GF_DTYPE_F16: return f(TypeTag<__half>{});
    case GF_DTYPE_BF16: return f(TypeTag<__nv_bfloat16>{});
    default:
        set_error("%s: unknown feature dtype %d (GF_DTYPE_F32 = 0, GF_DTYPE_F16 = 1, GF_DTYPE_BF16 = 2)", what, dtype);
        return GF_ERR_INVALID_ARG;
    }
}

// Four consecutive table values as fp32: one 16-byte load for float, one 8-byte load and two pair conversions for the
// 2-byte types.  The conversions are exact, so the arithmetic that follows is the fp32 arithmetic on the upcast table.
template <class T>
__device__ __forceinline__ float4 load4(const T *p);
template <>
__device__ __forceinline__ float4 load4<float>(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }
template <>
__device__ __forceinline__ float4 load4<__half>(const __half *p) {
    const uint2 raw = __ldg(reinterpret_cast<const uint2 *>(p));
    const float2 lo = __half22float2(*reinterpret_cast<const __half2 *>(&raw.x));
    const float2 hi = __half22float2(*reinterpret_cast<const __half2 *>(&raw.y));
    return make_float4(lo.x, lo.y, hi.x, hi.y);
}
template <>
__device__ __forceinline__ float4 load4<__nv_bfloat16>(const __nv_bfloat16 *p) {
    const uint2 raw = __ldg(reinterpret_cast<const uint2 *>(p));
    const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&raw.x));
    const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&raw.y));
    return make_float4(lo.x, lo.y, hi.x, hi.y);
}

// One table value as fp32 (the scalar loads of daf_kernel).
__device__ __forceinline__ float load1(const float *p) { return __ldg(p); }
__device__ __forceinline__ float load1(const __half *p) { return __half2float(__ldg(p)); }
__device__ __forceinline__ float load1(const __nv_bfloat16 *p) { return __bfloat162float(__ldg(p)); }

struct DafParams {
    gf_daf_desc d;
    const void *feat;         // [B, M, F, C] of the kernel's element type T
    const int32_t *shape;
    const int32_t *start;
    const float *loc;
    const float *weights;
    float *out;               // forward
    const float *grad_out;    // backward
    float *grad_feat, *grad_loc, *grad_weights;
};

struct DafFusedParams {
    gf_daf_desc d;
    int K;                        // key points per anchor
    const void *feat;             // [B, M, F, C] of the kernel's element type T
    const int32_t *shape;
    const int32_t *start;
    const float *loc;             // [B, A*K, M, 2]
    const float *logits;          // [B, A, K, M, L, Gr] raw (pre-softmax) weights
    const uint8_t *pmask;         // [B, A, K, M] or NULL
    const uint8_t *wmask;         // [B, A, K, M, L, Gr] or NULL
    float *out;                   // forward:  [B, A, C]
    float *stats;                 // forward writes / backward reads [B, A, Gr, 2] = (max*log2e, 1/sum)
    const float *out_saved;       // backward: the forward output
    const float *grad_out;        // backward: [B, A, C]
    float *grad_feat, *grad_loc, *grad_logits;
};

// What one launch of the sampling kernels computes.  kBackwardNoFeatGrad: the weight and location gradients alone, each
// summed in an order fixed by the inputs (no floating-point atomics); daf_det.cu gathers the feature gradient.
enum class DafPass { kForward, kBackward, kBackwardNoFeatGrad };

// daf.cu (dtype: GF_DTYPE_* of the feature table / maps, checked by the caller)
int launch_daf(const DafParams &p, int dtype, DafPass pass, int num_sms, cudaStream_t stream);
int launch_daf_format(const gf_daf_format_desc &d, int dtype, void *const *maps, void *table, bool inverse, cudaStream_t stream);
// daf_fused.cu
bool daf_fused_supported(const gf_daf_desc &d, int K);
int launch_daf_fused(const DafFusedParams &p, int dtype, DafPass pass, int num_sms, cudaStream_t stream);
// daf_det.cu: the ordered feature gradient of the deterministic backward (GF_BWD_DETERMINISTIC).
// daf_det_workspace_bytes: 0 with a message when the desc is outside the route's limits.  launch_daf_det_feat_grad
// adds (+=) the feature gradient of the plain op (fp = nullptr) or of the fused one (p = nullptr) into grad_feat.
size_t daf_det_workspace_bytes(const gf_daf_desc &d);
int launch_daf_det_feat_grad(const DafParams *p, const DafFusedParams *fp, void *workspace, int num_sms,
                             cudaStream_t stream);

struct PairSetup {     // 64 bytes per (camera, level) pair
    int row[4];        // element offset of each corner row inside the batch's feature block (row * C)
    float w[4];        // bilinear corner weights, 0 where the corner is outside the map
    float lh, lw;      // fractional parts (backward only)
    float fh, fw;      // level height / width as floats (backward only)
    int ok;            // bit k: corner k lies inside the map
    int cam;           // camera of this pair
    int pad0, pad1;
};

// Level table into shared memory (dynamically indexed registers would spill to local memory); ends with a
// __syncthreads, so every thread of the block must call it.
__device__ __forceinline__ void load_level_table(const gf_daf_desc &d, const int32_t *shape, const int32_t *start,
                                                 int *lh, int *lw, int *ls) {
    if (threadIdx.x < d.num_scale) {
        lh[threadIdx.x] = shape[2 * threadIdx.x];
        lw[threadIdx.x] = shape[2 * threadIdx.x + 1];
        ls[threadIdx.x] = start[threadIdx.x];
    }
    __syncthreads();
}

// ---- The sampling arithmetic of every DAF kernel: the camera gate, the bilinear cell with its corner weights and
// the fused op's softmax weight.  The deterministic backward (daf_det.cu) re-derives the cells and coefficients of the
// default kernels and is exact only while both evaluate the same expressions, so every kernel calls these functions
// instead of restating them.  nvcc contracts multiply/add pairs: operand order is part of each definition.

// Location (lx, ly) of point bp in camera m, and the gate: the camera sees the point strictly inside (0, 1)^2.
__device__ __forceinline__ bool cam_gate(const float *loc, long long bp, int M, int m, float &lx, float &ly) {
    lx = __ldg(loc + (bp * M + m) * 2); ly = __ldg(loc + (bp * M + m) * 2 + 1);
    return lx > 0.f && lx < 1.f && ly > 0.f && ly < 1.f;
}

// The bilinear cell of a location on an h x w map (pixel centres at +0.5): its unclamped top-left corner (y0, x0),
// the fractional parts lh, lw and their complements hh, hw.  Corner k is (y0 + k/2, x0 + k%2).
struct BilinearCell {
    int y0, x0;
    float lh, lw, hh, hw;
    __device__ __forceinline__ float weight(int k) const { return k == 0 ? hh * hw : k == 1 ? hh * lw : k == 2 ? lh * hw : lh * lw; }
    // row y0 + dy / column x0 + dx (dy, dx = 0 or 1) lies inside the h x w map, and so does corner k
    __device__ __forceinline__ bool row_inside(int dy, int h) const { return dy ? y0 + 1 <= h - 1 : y0 >= 0; }
    __device__ __forceinline__ bool col_inside(int dx, int w) const { return dx ? x0 + 1 <= w - 1 : x0 >= 0; }
    __device__ __forceinline__ bool inside(int k, int h, int w) const { return row_inside(k >> 1, h) && col_inside(k & 1, w); }
};

__device__ __forceinline__ BilinearCell bilinear_cell(float lx, float ly, int h, int w) {
    const float y_im = ly * static_cast<float>(h) - 0.5f, x_im = lx * static_cast<float>(w) - 0.5f;
    const float yf = floorf(y_im), xf = floorf(x_im), lh = y_im - yf, lw = x_im - xf;
    return {static_cast<int>(yf), static_cast<int>(xf), lh, lw, 1.f - lh, 1.f - lw};
}

// The scalar kernels' step (daf_kernel, daf_det_generic_kernel): the bilinear value of the corner values v (0 for
// corners outside the map) and its derivatives along x_im and y_im.
__device__ __forceinline__ float bilinear_value(const BilinearCell &c, const float v[4], float &dvx, float &dvy) {
    float val = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) val = fmaf(c.weight(k), v[k], val);
    dvx = fmaf(-c.hh, v[0], 0.f); dvx = fmaf(c.hh, v[1], dvx); dvx = fmaf(-c.lh, v[2], dvx); dvx = fmaf(c.lh, v[3], dvx);
    dvy = fmaf(-c.hw, v[0], 0.f); dvy = fmaf(-c.lw, v[1], dvy); dvy = fmaf(c.hw, v[2], dvy); dvy = fmaf(c.lw, v[3], dvy);
    return val;
}

// The fused op's softmax term exp2(logit * log2e - mlog) (mlog = the group's max * log2e), and the weight term / sum
// (inv = 1 / sum) of entry i, 0 where the weight mask wm (NULL: none) is off: a select, never a multiply, since a
// masked logit may be anything.
__device__ __forceinline__ float softmax_term(float logit, float mlog) { return ex2_approx(fmaf(logit, kLog2e, -mlog)); }
template <class I>
__device__ __forceinline__ float softmax_weight(float logit, float mlog, float inv, const uint8_t *wm, I i) {
    const float wt = softmax_term(logit, mlog) * inv;
    return (wm && !wm[i]) ? 0.f : wt;
}

__device__ __forceinline__ bool pair_setup(const gf_daf_desc &d, const float *loc, const int *lh, const int *lw, const int *ls,
                                           long long bp, int m, int lv, PairSetup &o) {
    const int M = d.num_cams, F = d.num_feat, C = d.num_embeds;
    float lx, ly;
    const bool gate = cam_gate(loc, bp, M, m, lx, ly);
    const int h = lh[lv], w = lw[lv];
    const BilinearCell cell = bilinear_cell(lx, ly, h, w);
    o.lh = cell.lh; o.lw = cell.lw;
    o.fh = static_cast<float>(h); o.fw = static_cast<float>(w);
    const bool oky0 = cell.row_inside(0, h), oky1 = cell.row_inside(1, h), okx0 = cell.col_inside(0, w), okx1 = cell.col_inside(1, w);
    const int cy0 = max(cell.y0, 0), cy1 = min(cell.y0 + 1, h - 1), cx0 = max(cell.x0, 0), cx1 = min(cell.x0 + 1, w - 1);
    const int base = m * F + ls[lv];
    o.row[0] = (base + cy0 * w + cx0) * C;
    o.row[1] = (base + cy0 * w + cx1) * C;
    o.row[2] = (base + cy1 * w + cx0) * C;
    o.row[3] = (base + cy1 * w + cx1) * C;
    o.w[0] = (oky0 && okx0) ? cell.weight(0) : 0.f;
    o.w[1] = (oky0 && okx1) ? cell.weight(1) : 0.f;
    o.w[2] = (oky1 && okx0) ? cell.weight(2) : 0.f;
    o.w[3] = (oky1 && okx1) ? cell.weight(3) : 0.f;
    o.ok = (oky0 && okx0 ? 1 : 0) | (oky0 && okx1 ? 2 : 0) | (oky1 && okx0 ? 4 : 0) | (oky1 && okx1 ? 8 : 0);
    o.cam = m;
    o.pad0 = o.pad1 = 0;
    return gate;
}

// Setup of sampling point bp: lane p < M*L writes the setup of its pair (my_cam, my_lv) into the warp's slots.
// Returns the ballot of the pairs whose camera sees the point and, with a point-mask row pm ([M] or nullptr),
// whose pm[camera] is set.  The whole warp must call it; the slots are complete on return.
__device__ __forceinline__ uint32_t setup_pairs(const gf_daf_desc &d, const float *loc, const int *lh, const int *lw,
                                                const int *ls, long long bp, int lane, int my_cam, int my_lv,
                                                const uint8_t *pm, PairSetup *mine) {
    bool gate = false;
    if (lane < d.num_cams * d.num_scale) {
        PairSetup ps;
        gate = pair_setup(d, loc, lh, lw, ls, bp, my_cam, my_lv, ps);
        if (pm) gate = gate && pm[my_cam] != 0;    // a masked point has weight 0 in every level and group
        mine[lane] = ps;
    }
    const uint32_t visible = __ballot_sync(0xffffffffu, gate);
    __syncwarp();
    return visible;
}

// Visits the visible pairs of one sampling point for the channel slice [c0, c0 + 4) of this lane.
//   featb / gfeatb : feature table (element type T) and fp32 feature gradient of the point's batch
//   grad_loc, bp, M: location gradient and the point's index; the row address (bp * M + camera) * 2 is formed
//                    only where the row is written, so no pointer stays live across the visit (backward)
//   weight(pr)     : aggregation weight of pair pr for this lane's group
//   weight_grad(pr, wt, gw) : called by the first lane of each group with the group's dL/d(weight) of pair pr
// Forward accumulates into acc; backward leaves acc alone.  The callers' callables capture by value: capturing
// the kernel's locals by reference compiles the plain backward to a different register allocation.
// FEAT_GRAD = false leaves the feature gradient out (the deterministic backward gathers it in daf_det.cu); the weight
// and location gradients are the same code either way.
template <bool BACKWARD, bool FEAT_GRAD, class T, class Weight, class WeightGrad>
__device__ __forceinline__ void visit_pairs(const PairSetup *mine, uint32_t visible, const T *featb, float *gfeatb,
                                            int c0, int lane, int lanes_per_group, float4 gout, float *grad_loc,
                                            long long bp, int M, float4 &acc, Weight weight, WeightGrad weight_grad) {
    float gx = 0.f, gy = 0.f;
    uint32_t todo = visible;
    while (todo) {
        const int pr = __ffs(todo) - 1;
        todo &= todo - 1;
        const int4 rows = *reinterpret_cast<const int4 *>(mine[pr].row);      // warp-uniform loads
        const float4 cw = *reinterpret_cast<const float4 *>(mine[pr].w);
        const float wt = weight(pr);
        const float4 v0 = load4(featb + rows.x + c0);
        const float4 v1 = load4(featb + rows.y + c0);
        const float4 v2 = load4(featb + rows.z + c0);
        const float4 v3 = load4(featb + rows.w + c0);
        if (!BACKWARD) {
            const float a0 = cw.x * wt, a1 = cw.y * wt, a2 = cw.z * wt, a3 = cw.w * wt;
            acc.x = fmaf(a0, v0.x, acc.x); acc.y = fmaf(a0, v0.y, acc.y); acc.z = fmaf(a0, v0.z, acc.z); acc.w = fmaf(a0, v0.w, acc.w);
            acc.x = fmaf(a1, v1.x, acc.x); acc.y = fmaf(a1, v1.y, acc.y); acc.z = fmaf(a1, v1.z, acc.z); acc.w = fmaf(a1, v1.w, acc.w);
            acc.x = fmaf(a2, v2.x, acc.x); acc.y = fmaf(a2, v2.y, acc.y); acc.z = fmaf(a2, v2.z, acc.z); acc.w = fmaf(a2, v2.w, acc.w);
            acc.x = fmaf(a3, v3.x, acc.x); acc.y = fmaf(a3, v3.y, acc.y); acc.z = fmaf(a3, v3.z, acc.z); acc.w = fmaf(a3, v3.w, acc.w);
        } else {
            const float4 fr = *reinterpret_cast<const float4 *>(&mine[pr].lh);
            const int2 okcam = *reinterpret_cast<const int2 *>(&mine[pr].ok);
            const int ok = okcam.x;
            // d(out)/d(feat corner) = corner weight * aggregation weight, for corners inside the map
            if (FEAT_GRAD) {
                float *gfb = gfeatb + c0;
                if (ok & 1) atomicAdd(reinterpret_cast<float4 *>(gfb + rows.x), make_float4(cw.x * wt * gout.x, cw.x * wt * gout.y, cw.x * wt * gout.z, cw.x * wt * gout.w));
                if (ok & 2) atomicAdd(reinterpret_cast<float4 *>(gfb + rows.y), make_float4(cw.y * wt * gout.x, cw.y * wt * gout.y, cw.y * wt * gout.z, cw.y * wt * gout.w));
                if (ok & 4) atomicAdd(reinterpret_cast<float4 *>(gfb + rows.z), make_float4(cw.z * wt * gout.x, cw.z * wt * gout.y, cw.z * wt * gout.z, cw.z * wt * gout.w));
                if (ok & 8) atomicAdd(reinterpret_cast<float4 *>(gfb + rows.w), make_float4(cw.w * wt * gout.x, cw.w * wt * gout.y, cw.w * wt * gout.z, cw.w * wt * gout.w));
            }
            // g . v_k for the four corners (outside corners carry weight 0; their clamped values are masked below)
            const float m0 = (ok & 1) ? 1.f : 0.f, m1 = (ok & 2) ? 1.f : 0.f, m2 = (ok & 4) ? 1.f : 0.f, m3 = (ok & 8) ? 1.f : 0.f;
            const float d0 = m0 * (gout.x * v0.x + gout.y * v0.y + gout.z * v0.z + gout.w * v0.w);
            const float d1 = m1 * (gout.x * v1.x + gout.y * v1.y + gout.z * v1.z + gout.w * v1.w);
            const float d2 = m2 * (gout.x * v2.x + gout.y * v2.y + gout.z * v2.z + gout.w * v2.w);
            const float d3 = m3 * (gout.x * v3.x + gout.y * v3.y + gout.z * v3.z + gout.w * v3.w);
            const float lhh = fr.x, lww = fr.y, hh = 1.f - lhh, hw = 1.f - lww;
            // d(out)/d(weight) = sampled value . g   (deformable_aggregation_cuda.cu:117-119)
            float gw = hh * hw * d0 + hh * lww * d1 + lhh * hw * d2 + lhh * lww * d3;
            // d(val)/d(x_im), d(val)/d(y_im)   (deformable_aggregation_cuda.cu:85-121)
            gx = fmaf(fr.w * wt, -hh * d0 + hh * d1 - lhh * d2 + lhh * d3, gx);
            gy = fmaf(fr.z * wt, -hw * d0 - lww * d1 + hw * d2 + lww * d3, gy);
#pragma unroll
            for (int o = 1; o < 32; o <<= 1)
                if (o < lanes_per_group) gw += __shfl_xor_sync(0xffffffffu, gw, o);
            if ((lane & (lanes_per_group - 1)) == 0) weight_grad(pr, wt, gw);
            // the location gradient of a camera is complete after its last visible level
            const int m = okcam.y;
            const bool cam_done = todo == 0 || mine[__ffs(todo) - 1].cam != m;
            if (cam_done) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    gx += __shfl_xor_sync(0xffffffffu, gx, o);
                    gy += __shfl_xor_sync(0xffffffffu, gy, o);
                }
                if (lane == 0) {
                    float *gl = grad_loc + (bp * M + m) * 2;
                    gl[0] += gx;
                    gl[1] += gy;
                }
                gx = 0.f; gy = 0.f;
            }
        }
    }
}

// conditions of the one-warp-per-point fast kernels: C % 128 == 0, a group = a power-of-two run of whole
// lanes, at most 32 (camera, level) pairs, 32-bit row offsets
inline bool daf_vec4_ok(const gf_daf_desc &d) {
    if (d.num_embeds % 128 != 0) return false;
    if (d.num_cams * d.num_scale > 32) return false;
    if (static_cast<long long>(d.num_cams) * d.num_feat * d.num_embeds >= (1ll << 31)) return false;
    const int gdim = d.num_embeds / d.num_groups;
    if (gdim % 4 != 0) return false;
    const int lpg = gdim / 4;
    return lpg <= 32 && (lpg & (lpg - 1)) == 0;
}

// CTAs for `items` warp-sized work items (points or anchors): one warp each, at most 64 CTAs per SM; the kernels
// loop over what does not fit
inline int daf_grid(long long items, int num_sms) {
    const int per_cta = kDafThreads / 32;
    const long long want = (items + per_cta - 1) / per_cta;
    const long long cap = static_cast<long long>(num_sms) * 64;
    return static_cast<int>(want < cap ? want : cap);
}

}  // namespace gf
