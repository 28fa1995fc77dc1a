// Key points of Gaussian anchors for the deformable aggregation (gf_daf_anchor_key_points / _backward):
// SparseGaussian3DKeyPointsGenerator.forward (model/encoder/gaussian_encoder/deformable_module.py:51-90) with
// get_rotation_matrix (model/utils/utils.py:20-69) and safe_sigmoid (model/utils/safe_ops.py:7-9), one thread per
// anchor, fp64 inside and one rounding per output.  For anchor row x (fp32, anchor_dim columns) and key point k:
//   sig(v)  = 1 / (1 + exp(-clamp(v, -9.21f, 9.21f)))
//   xyz     = lo + extent * sig(x[0:3]),   gs = scale_lo + scale_extent * sig(x[3:6])
//   s_k     = fix_scale[k] (k < Kf),   (sig(learnable_logits[k - Kf]) - 0.5) * learnable_fixed_scale (k >= Kf)
//   kp_k    = R(q)^T (s_k * gs) + xyz,   R = quat_rotation of q = x[6:10] (F.normalize first)
// The backward sums over k in ascending order in registers: no atomics, so the gradients are bit-reproducible.
#include "common.cuh"

namespace gf {

constexpr int kAnchorThreads = 64;            // 25 600 anchors -> 400 CTAs: every SM gets work

struct KpsArgs {
    gf_daf_kps_desc d;
    long long total;          // batch * num_anchors
    const float *anchor;      // [B, A, anchor_dim]
    const float *fix;         // [Kf, 3]
    const float *learn;       // [B, A, Kl, 3] or NULL when Kl == 0
};

// what every key point of one anchor shares
struct Frame {
    Sigmoid sx[3], sg[3];
    double xyz[3], gs[3];
    double q[4], R[3][3], inv_norm;
    bool below_eps;           // |q| < 1e-12f: F.normalize divided by the epsilon
};

__device__ __forceinline__ Frame anchor_frame(const KpsArgs &a, const float *row) {
    Frame f;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        f.sx[i] = safe_sigmoid(__ldg(row + i));
        f.sg[i] = safe_sigmoid(__ldg(row + 3 + i));
        f.xyz[i] = static_cast<double>(a.d.lo[i]) + static_cast<double>(a.d.extent[i]) * f.sx[i].s;
        f.gs[i] = static_cast<double>(a.d.scale_lo) + static_cast<double>(a.d.scale_extent) * f.sg[i].s;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) f.q[i] = __ldg(row + 6 + i);
    f.below_eps = quat_rotation(f.q, f.R, f.inv_norm) < kNormEps;
    return f;
}

// s_k of anchor `ba` for k in [0, Kf + Kl); sl receives the learnable sigmoids (untouched for a fixed point)
__device__ __forceinline__ void key_scale(const KpsArgs &a, long long ba, int k, double s[3], Sigmoid sl[3]) {
    const int Kf = a.d.num_fixed;
    if (k < Kf) {
#pragma unroll
        for (int j = 0; j < 3; ++j) s[j] = __ldg(a.fix + 3 * k + j);
    } else {
        const float *l = a.learn + (ba * a.d.num_learnable + (k - Kf)) * 3;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            sl[j] = safe_sigmoid(__ldg(l + j));
            s[j] = (sl[j].s - 0.5) * static_cast<double>(a.d.learnable_fixed_scale);
        }
    }
}

// one thread per (b, a): key_points[b, a, k, :] for every k
__global__ void __launch_bounds__(kAnchorThreads)
daf_anchor_kp_kernel(const KpsArgs a, float *__restrict__ key_points) {
    const long long ba = static_cast<long long>(blockIdx.x) * kAnchorThreads + threadIdx.x;
    if (ba >= a.total) return;
    const Frame f = anchor_frame(a, a.anchor + ba * a.d.anchor_dim);
    const int K = a.d.num_fixed + a.d.num_learnable;
    float *out = key_points + ba * K * 3;
    for (int k = 0; k < K; ++k) {
        double s[3];
        Sigmoid sl[3];
        key_scale(a, ba, k, s, sl);
        const double v[3] = {s[0] * f.gs[0], s[1] * f.gs[1], s[2] * f.gs[2]};
#pragma unroll
        for (int i = 0; i < 3; ++i)
            out[3 * k + i] = __double2float_rn(((f.R[0][i] * v[0] + f.R[1][i] * v[1]) + f.R[2][i] * v[2]) + f.xyz[i]);
    }
}

// one thread per (b, a), with g_k = grad_key_points[b, a, k, :] and v_k = s_k * gs:
//   dxyz = sum_k g_k,  dv_k = R g_k,  dgs = sum_k s_k * dv_k,  d(learnable s_k) = gs * dv_k,  dR = sum_k v_k g_k^T,
// then through quat_rotation_backward and the clamped sigmoids.  Columns 10.. of grad_anchor are written as 0.
__global__ void __launch_bounds__(kAnchorThreads)
daf_anchor_kp_grad_kernel(const KpsArgs a, const float *__restrict__ grad_kp, float *__restrict__ grad_anchor,
                          float *__restrict__ grad_learn) {
    const long long ba = static_cast<long long>(blockIdx.x) * kAnchorThreads + threadIdx.x;
    if (ba >= a.total) return;
    const Frame f = anchor_frame(a, a.anchor + ba * a.d.anchor_dim);
    const int Kf = a.d.num_fixed, K = Kf + a.d.num_learnable;
    const double lfs = a.d.learnable_fixed_scale;
    double dxyz[3] = {0.0, 0.0, 0.0}, dgs[3] = {0.0, 0.0, 0.0};
    double dR[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
    for (int k = 0; k < K; ++k) {
        double s[3];
        Sigmoid sl[3];
        key_scale(a, ba, k, s, sl);
        const float *gk = grad_kp + (ba * K + k) * 3;
        const double g[3] = {__ldg(gk), __ldg(gk + 1), __ldg(gk + 2)};
        double dv[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            dxyz[j] += g[j];
            dv[j] = (f.R[j][0] * g[0] + f.R[j][1] * g[1]) + f.R[j][2] * g[2];
            dgs[j] += s[j] * dv[j];
            const double v = s[j] * f.gs[j];
#pragma unroll
            for (int i = 0; i < 3; ++i) dR[j][i] += v * g[i];
        }
        if (k >= Kf) {
            float *gl = grad_learn + (ba * a.d.num_learnable + (k - Kf)) * 3;
#pragma unroll
            for (int j = 0; j < 3; ++j) gl[j] = __double2float_rn(f.gs[j] * dv[j] * lfs * sl[j].ds);
        }
    }
    float *ga = grad_anchor + ba * a.d.anchor_dim;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        ga[i] = __double2float_rn(dxyz[i] * static_cast<double>(a.d.extent[i]) * f.sx[i].ds);
        ga[3 + i] = __double2float_rn(dgs[i] * static_cast<double>(a.d.scale_extent) * f.sg[i].ds);
    }
    double dq[4];
    quat_rotation_backward(f.q, f.inv_norm, dR, dq, f.below_eps);
#pragma unroll
    for (int i = 0; i < 4; ++i) ga[6 + i] = __double2float_rn(dq[i]);
    for (int c = 10; c < a.d.anchor_dim; ++c) ga[c] = 0.f;
}

// the checks both entry points share; *work = B * A (threads to launch)
static int check_kps(const gf_daf_kps_desc *d, const float *anchor, const float *fix_scale,
                     const float *learnable_logits, const char *what, long long *work) {
    GF_REQUIRE(d != nullptr, GF_ERR_INVALID_ARG, "%s: desc is NULL", what);
    GF_REQUIRE(d->batch >= 0 && d->num_anchors >= 0 && d->anchor_dim >= 0 && d->num_fixed >= 0 && d->num_learnable >= 0,
               GF_ERR_INVALID_ARG, "%s: negative size (batch=%d, num_anchors=%d, anchor_dim=%d, num_fixed=%d, "
               "num_learnable=%d)", what, d->batch, d->num_anchors, d->anchor_dim, d->num_fixed, d->num_learnable);
    GF_REQUIRE(d->anchor_dim >= 10, GF_ERR_INVALID_ARG,
               "%s: anchor_dim=%d, the anchor needs at least 10 columns (xyz, scale, rotation)", what, d->anchor_dim);
    const long long ba = static_cast<long long>(d->batch) * d->num_anchors;
    const long long K = static_cast<long long>(d->num_fixed) + d->num_learnable;
    GF_REQUIRE(ba < (1ll << 31) && ba * K < (1ll << 31) && ba * d->anchor_dim < (1ll << 31), GF_ERR_UNSUPPORTED,
               "%s: batch * num_anchors * (num_fixed + num_learnable) = %lld * %lld and batch * num_anchors * "
               "anchor_dim must stay below 2^31", what, ba, K);
    *work = ba;
    if (ba == 0) return GF_OK;
    GF_REQUIRE(K > 0, GF_ERR_INVALID_ARG, "%s: num_fixed + num_learnable is 0", what);
    GF_REQUIRE(anchor != nullptr, GF_ERR_INVALID_ARG, "%s: anchor is NULL", what);
    if (d->num_fixed > 0) GF_REQUIRE(fix_scale != nullptr, GF_ERR_INVALID_ARG, "%s: fix_scale is NULL", what);
    if (d->num_learnable > 0)
        GF_REQUIRE(learnable_logits != nullptr, GF_ERR_INVALID_ARG, "%s: learnable_logits is NULL", what);
    return GF_OK;
}

static KpsArgs kps_args(const gf_daf_kps_desc *d, long long total, const float *anchor, const float *fix_scale,
                        const float *learnable_logits) {
    KpsArgs a;
    a.d = *d; a.total = total;
    a.anchor = anchor; a.fix = fix_scale; a.learn = learnable_logits;
    return a;
}

static unsigned anchor_blocks(long long total) {
    return static_cast<unsigned>((total + kAnchorThreads - 1) / kAnchorThreads);
}

}  // namespace gf

using namespace gf;

extern "C" {

int gf_daf_anchor_key_points(const gf_daf_kps_desc *desc, const float *anchor, const float *fix_scale,
                             const float *learnable_logits, float *key_points, gf_stream_t stream_) {
    long long total = 0;
    int rc = check_kps(desc, anchor, fix_scale, learnable_logits, "daf anchor key points", &total);
    if (rc != GF_OK) return rc;
    if (total == 0) return GF_OK;
    GF_REQUIRE(key_points != nullptr, GF_ERR_INVALID_ARG, "daf anchor key points: key_points is NULL");
    const KpsArgs a = kps_args(desc, total, anchor, fix_scale, learnable_logits);
    daf_anchor_kp_kernel<<<anchor_blocks(total), kAnchorThreads, 0, static_cast<cudaStream_t>(stream_)>>>(a, key_points);
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}

int gf_daf_anchor_key_points_backward(const gf_daf_kps_desc *desc, const float *anchor, const float *fix_scale,
                                      const float *learnable_logits, const float *grad_key_points,
                                      float *grad_anchor, float *grad_learnable, gf_stream_t stream_) {
    long long total = 0;
    int rc = check_kps(desc, anchor, fix_scale, learnable_logits, "daf anchor key points backward", &total);
    if (rc != GF_OK) return rc;
    if (total == 0) return GF_OK;
    GF_REQUIRE(grad_key_points != nullptr, GF_ERR_INVALID_ARG,
               "daf anchor key points backward: grad_key_points is NULL");
    GF_REQUIRE(grad_anchor != nullptr, GF_ERR_INVALID_ARG, "daf anchor key points backward: grad_anchor is NULL");
    if (desc->num_learnable > 0)
        GF_REQUIRE(grad_learnable != nullptr, GF_ERR_INVALID_ARG,
                   "daf anchor key points backward: grad_learnable is NULL");
    const KpsArgs a = kps_args(desc, total, anchor, fix_scale, learnable_logits);
    daf_anchor_kp_grad_kernel<<<anchor_blocks(total), kAnchorThreads, 0, static_cast<cudaStream_t>(stream_)>>>(
        a, grad_key_points, grad_anchor, grad_learnable);
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}

}  // extern "C"
