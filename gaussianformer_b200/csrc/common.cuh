// Shared device/host helpers for the sm_90a kernels (splat + deformable aggregation).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "gf_b200.h"

namespace gf {

// ---------------------------------------------------------------------------------------------
// error plumbing (host)
// ---------------------------------------------------------------------------------------------
void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what);

#define GF_CUDA_TRY(expr)                                         \
    do {                                                          \
        cudaError_t _e = (expr);                                  \
        if (_e != cudaSuccess) return ::gf::cuda_fail(_e, #expr); \
    } while (0)

#define GF_REQUIRE(cond, code, ...)      \
    do {                                 \
        if (!(cond)) {                   \
            ::gf::set_error(__VA_ARGS__); \
            return (code);               \
        }                                \
    } while (0)

// The class counts C the splat kernels are compiled for.  dispatch_classes returns f(std::integral_constant<int, C>{})
// for one of them; any other C is reported as `what`'s error.
constexpr int kMinClasses = 16, kMaxClasses = 20;
template <int CC = kMinClasses, class F>
int dispatch_classes(int C, const char *what, F &&f) {
    if constexpr (CC > kMaxClasses) {
        set_error("%s: class count C=%d is not compiled in (supported: %d..%d)", what, C, kMinClasses, kMaxClasses);
        return GF_ERR_UNSUPPORTED;
    } else {
        if (C == CC) return f(std::integral_constant<int, CC>{});
        return dispatch_classes<CC + 1>(C, what, f);
    }
}

// ---------------------------------------------------------------------------------------------
// geometry of the splat pipeline
// ---------------------------------------------------------------------------------------------
constexpr int kBinX = 8;        // render CTA footprint in columns: 8 (x) by 4 (y) ...
constexpr int kBinY = 4;
constexpr int kBinZ = 16;       // ... by 16 voxels in z (one z-chunk)
constexpr int kRenderThreads = 128;
constexpr int kGeomFloats = 12; // mu(3) k(1) c6(6) pad(2)

__host__ __device__ constexpr int round_up(int v, int m) { return (v + m - 1) / m * m; }
// one record = geometry + class vector, padded to a whole number of 128-byte lines.  Forward records (render kernels), as
// 16-byte chunks: 0 = mu(3), amplitude (base variant: z-level mask of the box) | 1 = exponent coefficients a b c d |
// 2 = e f, classes 16 17 | 3..6 = classes 0..15 | 7 = classes 18 19, pad(2).  Classes 16 and 17 share the chunk of the
// last two coefficients so that an 18-class step is six 16-byte shared loads instead of five and two 8-byte ones.  The raw
// records of the backward keep the plain order: chunk 2 = e f 0 0, chunks 3..7 = classes 0..19.
__host__ __device__ constexpr int rec_floats(int C) { return round_up(kGeomFloats + round_up(C, 4), 32); }

// Integer box of one Gaussian, inclusive bounds packed lo | hi << 16 per axis; w = 1 when the
// clipped box is empty.  (reference: getRect, model/head/localagg/src/auxiliary.h:8-20)
struct __align__(16) PackedBox {
    uint32_t x, y, z, empty;
};

// The forward workspace of the splat pipeline (also the forward-style block of the backward workspace).  Only
// plan_forward_workspace (splat_prep.cu) decides its layout; kernels receive it whole and narrow it to one sample with
// sample_ws and number supertiles with supertile_of.
struct SplatWorkspace {
    uint32_t *flags;       // status block, 256 bytes: word 0 status bits, words 4..19 GF_RENDER_TIMING cycle counters
    uint32_t *pack_flags;  // [batch * pack_ctas] per-CTA error bits of the pack kernel
    float *records;        // [G, rec] per sample
    PackedBox *boxes;      // [G] per sample
    uint32_t *masks;       // [nsuper, nwords] per sample: bit g of supertile s: box(g) overlaps s
    int32_t *lists;        // [nsuper, G] per sample: ascending Gaussian indices per supertile
    int32_t *counts;       // [nsuper] per sample
    int rec;               // floats per record: rec_floats(C)
    int st;                // supertile edge (columns), a power of two
    int nsx, nsy, nsuper;  // supertile grid
    int nwords;            // ceil(G/32)
    int pack_ctas;         // pack CTAs per sample
    int batch;             // samples
};

__host__ __device__ inline int batch_of(const gf_splat_desc &d) { return d.batch > 0 ? d.batch : 1; }

constexpr int kPackThreads = 64;   // small CTAs: ~400 of them cover the 132 SMs several times over

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__
// Launches `kernel` so that it may become resident while the preceding kernel of the stream is still
// running (programmatic stream serialization).  The kernel must call pdl_wait() before it touches
// anything the preceding kernel writes.
template <class... Params>
cudaError_t launch_chained(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, const Params &...p) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, p...);
}


__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Lane-wise fp32 pair arithmetic.  sm_90 has no packed fp32 instructions, so each is two scalar operations; the
// explicit _rn forms keep the compiler from contracting a multiply and an add, so every lane rounds as written.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, 0x4000;\n"   // suspend-time hint (ns): sleep, don't poll
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return done != 0;
}
// Bounded spin: a protocol bug must surface as a launch failure (trap), never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 24)) __trap();
    }
}
// Programmatic dependent launch (the three kernels of a forward call are chained with it, see
// launch_chained): launch_dependents lets the next kernel of the stream become resident while this grid
// is still running; wait blocks until the preceding grid has completed and its writes are visible.
// Both are no-ops for a kernel launched without the attribute / without a dependent.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// Phase A of the bin kernels (render_tile_kernel, backward_bin_kernel): the bin's ordered Gaussian list, resolved from
// its supertile's list.  A bin entry is one Gaussian whose box overlaps the bin: .x holds the box clipped to the bin as
// bit masks -- x columns in bits 0-7, y columns in bits 8-11, z levels in bits 16-31 -- and .y the Gaussian index.
// All NT threads of the CTA test the candidates cand[cpos..ncand), the ascending list of supertile s of the sample `ws`
// is narrowed to, fetching kPre rounds of NT before testing any (memory-level parallelism), and append the survivors to
// `list` in the same order, compacted with ballots, until the candidates run out or another round might overflow SEG
// entries.  Advances cpos past the tested candidates and returns the number of entries.
template <int NT, int kPre, int SEG>
__device__ __forceinline__ int resolve_bin_list(const gf_splat_desc &d, const SplatWorkspace &ws, int s, int ncand, int &cpos,
                                                int binX0, int binY0, int binZ0, uint2 *list, int (&warp_count)[2][NT / 32]) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int32_t *cand = ws.lists + static_cast<size_t>(s) * d.G;
    const PackedBox *boxes = ws.boxes;
    const uint32_t bX1 = min(binX0 + kBinX, d.H) - 1, bY1 = min(binY0 + kBinY, d.W) - 1, bZ1 = min(binZ0 + kBinZ, d.D) - 1;
    int nlist = 0;
    while (cpos < ncand && nlist + NT <= SEG) {
        int gg[kPre];
        uint4 bb[kPre];
#pragma unroll
        for (int u = 0; u < kPre; ++u) {
            const int i = cpos + u * NT + tid;
            gg[u] = i < ncand ? __ldg(cand + i) : -1;
        }
#pragma unroll
        for (int u = 0; u < kPre; ++u)
            bb[u] = gg[u] >= 0 ? __ldg(reinterpret_cast<const uint4 *>(boxes) + gg[u]) : make_uint4(1u, 1u, 1u, 1u);
#pragma unroll
        for (int u = 0; u < kPre; ++u) {
            if (cpos >= ncand || nlist + NT > SEG) break;   // uniform
            const uint4 b = bb[u];
            const uint32_t x0 = b.x & 0xffffu, x1 = b.x >> 16, y0 = b.y & 0xffffu, y1 = b.y >> 16,
                           z0 = b.z & 0xffffu, z1 = b.z >> 16;
            const bool hit = gg[u] >= 0 && x0 <= bX1 && x1 >= static_cast<uint32_t>(binX0) && y0 <= bY1 &&
                             y1 >= static_cast<uint32_t>(binY0) && z0 <= bZ1 && z1 >= static_cast<uint32_t>(binZ0) &&
                             b.w == 0u;
            const int rx0 = max(static_cast<int>(x0) - binX0, 0), rx1 = min(static_cast<int>(x1) - binX0, kBinX - 1);
            const int ry0 = max(static_cast<int>(y0) - binY0, 0), ry1 = min(static_cast<int>(y1) - binY0, kBinY - 1);
            const int rz0 = max(static_cast<int>(z0) - binZ0, 0), rz1 = min(static_cast<int>(z1) - binZ0, kBinZ - 1);
            const uint32_t xm = ((2u << rx1) - 1u) & ~((1u << rx0) - 1u);
            const uint32_t ym = ((2u << ry1) - 1u) & ~((1u << ry0) - 1u);
            const uint32_t zm = ((2u << rz1) - 1u) & ~((1u << rz0) - 1u);
            const uint2 entry = make_uint2(xm | (ym << 8) | (zm << 16), static_cast<uint32_t>(gg[u]));
            const uint32_t ballot = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) warp_count[u & 1][warp] = __popc(ballot);
            __syncthreads();
            int off = nlist, total = 0;
#pragma unroll
            for (int k = 0; k < NT / 32; ++k) {
                const int c = warp_count[u & 1][k];
                if (k < warp) off += c;
                total += c;
            }
            if (hit) list[off + __popc(ballot & lanemask_lt())] = entry;
            nlist += total;
            cpos += NT;
        }
        __syncthreads();
    }
    return nlist;
}

// ((v - origin) / cell) truncated toward zero, with the exact fp32 operation order of
// `((x - pc_min) / grid_size).to(torch.int)` (local_aggregate/__init__.py:137,139).
__device__ __forceinline__ int voxel_coord(float v, float origin, float cell) {
    return static_cast<int>(__fdiv_rn(__fsub_rn(v, origin), cell));
}

// Integer box of Gaussian g (inclusive bounds, clipped to the grid) and the error bits the
// reference asserts on.  Fuses the Python host preparation (trunc voxel index of the mean, ceil
// radius; local_aggregate/__init__.py:139-142, prob: :151-153, prob_fast: :151) with getRect
// (src/auxiliary.h:8-20).  Returns true when the clipped box is empty.
__device__ __forceinline__ bool gaussian_box(const gf_splat_desc &d, const gf_splat_inputs &in, int g,
                                             const float mu[3], int lo[3], int hi[3], uint32_t &err) {
    const int dims[3] = {d.H, d.W, d.D};
    int m[3], r[3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
        m[a] = in.means_int ? in.means_int[3 * g + a] : voxel_coord(mu[a], d.pc_min[a], d.grid_size);
    if (in.radii) {
#pragma unroll
        for (int a = 0; a < 3; ++a) r[a] = (d.radii_axes == 3) ? in.radii[3 * g + a] : in.radii[g];
    } else {
        const float s[3] = {in.scales[3 * g], in.scales[3 * g + 1], in.scales[3 * g + 2]};
        if (d.radii_axes == 3) {
#pragma unroll
            for (int a = 0; a < 3; ++a)
                r[a] = static_cast<int>(ceilf(__fdiv_rn(__fmul_rn(s[a], d.scale_multiplier), d.grid_size)));
        } else {
            const float smax = fmaxf(s[0], fmaxf(s[1], s[2]));
            r[0] = r[1] = r[2] = static_cast<int>(ceilf(__fdiv_rn(__fmul_rn(smax, d.scale_multiplier), d.grid_size)));
        }
        if (d.radii_min > 0) {
#pragma unroll
            for (int a = 0; a < 3; ++a) r[a] = max(r[a], d.radii_min);
        }
    }
    bool empty = false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (m[a] < 0 || m[a] >= dims[a]) err |= GF_FLAG_MEAN_OUT_OF_GRID;
        if (r[a] < 1) err |= GF_FLAG_RADIUS_LT_1;
        // inclusive form of [min(dim,max(0,m-r)), min(dim,max(0,m+r+1)))
        const long long l = static_cast<long long>(m[a]) - r[a];
        const long long h = static_cast<long long>(m[a]) + r[a];
        lo[a] = static_cast<int>(l < 0 ? 0 : l);
        hi[a] = static_cast<int>(h > dims[a] - 1 ? dims[a] - 1 : h);
        if (l > dims[a] - 1 || h < 0 || lo[a] > hi[a]) empty = true;
    }
    return empty;
}

// ---- batch: the tensors of sample b (dense strides; NULL stays NULL; pts may be shared by the batch) ----------------
template <class T>
__device__ __forceinline__ T *adv(T *p, long long off) { return p ? p + off : p; }

__device__ __forceinline__ gf_splat_inputs sample_inputs(const gf_splat_desc &d, const gf_splat_inputs &in, int b) {
    gf_splat_inputs o;
    const long long G = d.G, N = d.N;
    const long long np = d.pts_shared ? 0 : b * N * 3;
    o.pts = adv(in.pts, np);
    o.points_int = adv(in.points_int, np);
    o.means = adv(in.means, b * G * 3);
    o.means_int = adv(in.means_int, b * G * 3);
    o.opacities = adv(in.opacities, b * G);
    o.semantics = adv(in.semantics, b * G * d.C);
    o.cov = adv(in.cov, b * G * d.cov_stride);
    o.radii = adv(in.radii, b * G * (d.radii_axes == 3 ? 3 : 1));
    o.scales = adv(in.scales, b * G * 3);
    o.rotations = adv(in.rotations, b * G * 4);
    return o;
}

// The workspace blocks of sample b: records, boxes, masks, lists and counts.  flags and pack_flags stay batch-level.
__device__ __forceinline__ SplatWorkspace sample_ws(const SplatWorkspace &ws, int G, int b) {
    SplatWorkspace o = ws;
    o.records = ws.records + static_cast<size_t>(b) * G * ws.rec;
    o.boxes = ws.boxes + static_cast<size_t>(b) * G;
    o.masks = ws.masks + static_cast<size_t>(b) * ws.nsuper * ws.nwords;
    o.lists = ws.lists + static_cast<size_t>(b) * ws.nsuper * G;
    o.counts = ws.counts + static_cast<size_t>(b) * ws.nsuper;
    return o;
}

// Supertile of column (x, y) (x, y >= 0): supertiles are st x st columns, numbered x-major.
__device__ __forceinline__ int supertile_of(const SplatWorkspace &ws, int x, int y) {
    const int sh = 31 - __clz(ws.st);
    return (x >> sh) * ws.nsy + (y >> sh);
}

__device__ __forceinline__ gf_splat_outputs sample_outputs(const gf_splat_desc &d, const gf_splat_outputs &out, int b, int ce_rows) {
    gf_splat_outputs o;
    const long long N = d.N;
    o.logits = adv(out.logits, b * N * d.C);
    o.bin_logits = adv(out.bin_logits, b * N);
    o.density = adv(out.density, b * N);
    o.probability = adv(out.probability, b * N);
    o.argmax = adv(out.argmax, b * N);
    o.logits_cn = adv(out.logits_cn, b * N * d.C);
    o.labels = adv(out.labels, b * N);
    o.class_weights = out.class_weights;
    o.ce_partials = adv(out.ce_partials, 2ll * b * ce_rows);
    return o;
}

__device__ __forceinline__ gf_splat_grads sample_grads(const gf_splat_desc &d, const gf_splat_grads &gr, int b) {
    gf_splat_grads o;
    const long long G = d.G, N = d.N;
    o.logits_grad = adv(gr.logits_grad, b * N * d.C);
    o.bin_logits_grad = adv(gr.bin_logits_grad, b * N);
    o.density_grad = adv(gr.density_grad, b * N);
    o.logits = adv(gr.logits, b * N * d.C);
    o.bin_logits = adv(gr.bin_logits, b * N);
    o.probability = adv(gr.probability, b * N);
    o.means_grad = adv(gr.means_grad, b * G * 3);
    o.opacity_grad = adv(gr.opacity_grad, b * G);
    o.semantics_grad = adv(gr.semantics_grad, b * G * d.C);
    o.cov_grad = adv(gr.cov_grad, b * G * d.cov_stride);
    o.scales_grad = adv(gr.scales_grad, b * G * 3);
    o.rotations_grad = adv(gr.rotations_grad, b * G * 4);
    return o;
}

// The scalar-type overloads the quaternion maps below are written with (float: the splat, double: the key-point
// generator of daf_anchor.cu).
__device__ __forceinline__ float q_sqrt(float v) { return sqrtf(v); }
__device__ __forceinline__ double q_sqrt(double v) { return sqrt(v); }
__device__ __forceinline__ float q_max(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ double q_max(double a, double b) { return fmax(a, b); }
__device__ __forceinline__ float q_div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double q_div(double a, double b) { return __ddiv_rn(a, b); }

// Rotation matrix of the NORMALISED quaternion (w,x,y,z) -- get_rotation_matrix, model/utils/utils.py:20-66
// (F.normalize: q / max(|q|, 1e-12), the epsilon as an fp32 tensor holds it).  R[k][l], row-major.  Returns |q|.
template <class T>
__device__ __forceinline__ T quat_rotation(const T q[4], T R[3][3], T &inv_norm) {
    const T n = q_sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    inv_norm = q_div(T(1), q_max(n, static_cast<T>(1e-12f)));
    const T w = q[0] * inv_norm, x = q[1] * inv_norm, y = q[2] * inv_norm, z = q[3] * inv_norm;
    R[0][0] = w * w + x * x - y * y - z * z; R[0][1] = T(2) * (x * y - w * z);         R[0][2] = T(2) * (x * z + w * y);
    R[1][0] = T(2) * (x * y + w * z);         R[1][1] = w * w - x * x + y * y - z * z; R[1][2] = T(2) * (y * z - w * x);
    R[2][0] = T(2) * (x * z - w * y);         R[2][1] = T(2) * (y * z + w * x);         R[2][2] = w * w - x * x - y * y + z * z;
    return n;
}

// The gradient of quat_rotation: dq (w.r.t. the UN-normalised q) from M = dL/dR, through the quaternion -> matrix map and
// F.normalize.  inv_norm is quat_rotation's.  below_eps: |q| < 1e-12, where F.normalize divides by the constant epsilon,
// so the gradient is M's pulled back and scaled, without the projection onto the sphere's tangent.
template <class T>
__device__ __forceinline__ void quat_rotation_backward(const T q[4], T inv_norm, const T M[3][3], T dq[4],
                                                       bool below_eps) {
    const T w = q[0] * inv_norm, x = q[1] * inv_norm, y = q[2] * inv_norm, z = q[3] * inv_norm;
    const T gw = T(2) * (w * (M[0][0] + M[1][1] + M[2][2]) - z * M[0][1] + y * M[0][2] + z * M[1][0] - x * M[1][2] - y * M[2][0] + x * M[2][1]);
    const T gx = T(2) * (x * (M[0][0] - M[1][1] - M[2][2]) + y * M[0][1] + z * M[0][2] + y * M[1][0] - w * M[1][2] + z * M[2][0] + w * M[2][1]);
    const T gy = T(2) * (y * (-M[0][0] + M[1][1] - M[2][2]) + x * M[0][1] + w * M[0][2] + x * M[1][0] + z * M[1][2] - w * M[2][0] + z * M[2][1]);
    const T gz = T(2) * (z * (-M[0][0] - M[1][1] + M[2][2]) - w * M[0][1] + x * M[0][2] + w * M[1][0] + y * M[1][2] + x * M[2][0] + y * M[2][1]);
    const T dot = below_eps ? T(0) : w * gw + x * gx + y * gy + z * gz;
    dq[0] = inv_norm * (gw - w * dot);
    dq[1] = inv_norm * (gx - x * dot);
    dq[2] = inv_norm * (gy - y * dot);
    dq[3] = inv_norm * (gz - z * dot);
}

// safe_sigmoid (model/utils/safe_ops.py:7-9) in fp64, for the key-point generator (daf_anchor.cu) and the refinement
// (gaussian_refine.cu).  The constants are the values the reference's fp32 tensors hold.
constexpr double kLogitClamp = static_cast<double>(9.21f);   // safe_sigmoid's bound
constexpr double kNormEps = static_cast<double>(1e-12f);     // F.normalize's epsilon

struct Sigmoid {
    double s;    // sigmoid of the clamped logit
    double ds;   // its derivative w.r.t. the logit: s (1 - s) inside the clamp, bounds included; 0 outside (and NaN)
};

__device__ __forceinline__ Sigmoid safe_sigmoid(double x) {
    const double c = x < -kLogitClamp ? -kLogitClamp : (x > kLogitClamp ? kLogitClamp : x);   // NaN stays NaN
    const double s = 1.0 / (1.0 + exp(-c));
    return {s, (x >= -kLogitClamp && x <= kLogitClamp) ? s * (1.0 - s) : 0.0};
}

// Sigma^-1 = R^T diag(1/s^2) R as (xx,yy,zz,xy,yz,xz): the closed form of GaussianHead.prepare_gaussian_args'
// Cov = (S R)^T (S R); Cov.cpu().inverse() (model/head/gaussian_head.py:111-119), R orthogonal.
__device__ __forceinline__ void cov6_from_srt(const float s[3], const float q[4], float c6[6]) {
    float R[3][3], inv_norm;
    quat_rotation(q, R, inv_norm);
    const float d0 = __fdiv_rn(1.f, s[0] * s[0]), d1 = __fdiv_rn(1.f, s[1] * s[1]), d2 = __fdiv_rn(1.f, s[2] * s[2]);
    auto a = [&](int i, int j) { return R[0][i] * d0 * R[0][j] + R[1][i] * d1 * R[1][j] + R[2][i] * d2 * R[2][j]; };
    c6[0] = a(0, 0); c6[1] = a(1, 1); c6[2] = a(2, 2); c6[3] = a(0, 1); c6[4] = a(1, 2); c6[5] = a(0, 2);
}

// the six inverse-covariance entries (xx,yy,zz,xy,yz,xz) of Gaussian g (in: the tensors of ONE sample)
__device__ __forceinline__ void load_cov6_in(const gf_splat_desc &d, const gf_splat_inputs &in, int g, float c6[6]) {
    if (in.cov == nullptr) {
        const float s[3] = {__ldg(in.scales + 3 * g), __ldg(in.scales + 3 * g + 1), __ldg(in.scales + 3 * g + 2)};
        const float q[4] = {__ldg(in.rotations + 4 * g), __ldg(in.rotations + 4 * g + 1), __ldg(in.rotations + 4 * g + 2),
                            __ldg(in.rotations + 4 * g + 3)};
        cov6_from_srt(s, q, c6);
        return;
    }
    const float *cv = in.cov + static_cast<size_t>(g) * d.cov_stride;
    if (d.cov_stride == 9) {  // flat entries [0,4,8,1,5,2] of the row-major 3x3 (__init__.py:143)
        c6[0] = __ldg(cv); c6[1] = __ldg(cv + 4); c6[2] = __ldg(cv + 8); c6[3] = __ldg(cv + 1); c6[4] = __ldg(cv + 5); c6[5] = __ldg(cv + 2);
    } else {
#pragma unroll
        for (int i = 0; i < 6; ++i) c6[i] = __ldg(cv + i);
    }
}

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kKappa = 0.06349363593424097f;  // powf(2 * 3.1415926535f, -1.5f), localagg_prob/src/forward.cu:78

#endif  // __CUDACC__

}  // namespace gf
