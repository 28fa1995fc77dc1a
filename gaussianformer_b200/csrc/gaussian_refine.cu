// Gaussian refinement (gf_gaussian_refine / _backward): the arithmetic of SparseGaussian3DRefinementModule.forward
// (model/encoder/gaussian_encoder/refine_module.py:72-123) and SparseGaussian3DRefinementModuleV2.forward
// (refine_module_v2.py:64-108) after their MLP, one thread per anchor, fp64 inside and one rounding per output.  The
// contract, with every constant, is in include/gf_b200.h.  The backward recomputes the forward from out and anchor and
// writes every gradient entry of its row from registers: no atomics, so the gradients are bit-reproducible.
#include "common.cuh"

namespace gf {

constexpr int kRefineThreads = 64;                  // 25 600 anchors -> 400 CTAs: every SM gets work
constexpr int kMaxSem = GF_REFINE_MAX_SEMANTICS;
// safe_inverse_sigmoid's clamp (safe_ops.py:11-13) as an fp32 tensor holds its bounds: 1 - 0.9999 and 0.9999
constexpr double kInvLo = static_cast<double>(static_cast<float>(1.0 - 0.9999));
constexpr double kInvHi = static_cast<double>(0.9999f);
constexpr double kSoftplusThreshold = 20.0;         // F.softplus: x itself where x > 20

struct RefineArgs {
    gf_refine_desc d;
    long long total;          // batch * num_anchors
    const float *out;         // [B, A, out_dim]
    const float *anchor;      // [B, A, anchor_dim]
};

// what the outputs of one anchor share: o[0:10] of the header (V1 after the restriction and the residual add; V2
// [axyz, out[3:10]]) and the sigmoids and clamps on the way
struct Frame {
    double o[10];
    Sigmoid sm[3];            // ssig(o[0:3]): the means
    Sigmoid ss[3];            // ssig(o[3:6]): the scales
    Sigmoid sr[3];            // ssig(out[0:3]): V1 with restrict_xyz, V2's delta
    Sigmoid sa[3];            // V2: ssig(anchor[0:3])
    double orig[3], delta[3]; // V2
    double tc[3];             // V2: the clamped (orig + delta - lo) / extent
    bool tin[3];              // V2: ... inside the clamp, bounds included
    double rot[4], inv_norm;
    bool below_eps;           // |o[6:10]| < 1e-12f: F.normalize divided by the epsilon
};

// column j of the refined row for j >= 10 (the opacity and semantic logits; V1 adds the anchor's column inside the
// prefix, V2 has no prefix)
__device__ __forceinline__ double column(const RefineArgs &a, const float *row, const float *arow, int j) {
    const double v = __ldg(row + j);
    return j < a.d.refine_prefix ? v + static_cast<double>(__ldg(arow + j)) : v;
}

__device__ __forceinline__ Frame refine_frame(const RefineArgs &a, const float *row, const float *arow) {
    const gf_refine_desc &d = a.d;
    Frame f;
#pragma unroll
    for (int i = 0; i < 10; ++i) f.o[i] = __ldg(row + i);
    if (d.variant == GF_REFINE_V1) {
        if (d.restrict_xyz) {
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                f.sr[i] = safe_sigmoid(f.o[i]);
                f.o[i] = (2.0 * f.sr[i].s - 1.0) * static_cast<double>(d.unit[i]);
            }
        }
#pragma unroll
        for (int i = 0; i < 10; ++i)
            if (i < d.refine_prefix) f.o[i] += static_cast<double>(__ldg(arow + i));
    } else {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const double lo = d.lo[i], ext = d.extent[i];
            f.sr[i] = safe_sigmoid(f.o[i]);
            f.delta[i] = (2.0 * f.sr[i].s - 1.0) * static_cast<double>(d.unit[i]);
            f.sa[i] = safe_sigmoid(static_cast<double>(__ldg(arow + i)));
            f.orig[i] = f.sa[i].s * ext + lo;
            const double t = ((f.orig[i] + f.delta[i]) - lo) / ext;
            f.tin[i] = t >= kInvLo && t <= kInvHi;
            f.tc[i] = t < kInvLo ? kInvLo : (t > kInvHi ? kInvHi : t);   // NaN stays NaN
            f.o[i] = log(f.tc[i] / (1.0 - f.tc[i]));
        }
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        f.sm[i] = safe_sigmoid(f.o[i]);
        f.ss[i] = safe_sigmoid(f.o[3 + i]);
    }
    const double n = sqrt(f.o[6] * f.o[6] + f.o[7] * f.o[7] + f.o[8] * f.o[8] + f.o[9] * f.o[9]);
    f.inv_norm = 1.0 / fmax(n, kNormEps);
    f.below_eps = n < kNormEps;
#pragma unroll
    for (int i = 0; i < 4; ++i) f.rot[i] = f.o[6 + i] * f.inv_norm;
    return f;
}

__device__ __forceinline__ double grad_at(const float *g, long long i) {
    return g != nullptr ? static_cast<double>(__ldg(g + i)) : 0.0;
}

// one thread per (b, a)
__global__ void __launch_bounds__(kRefineThreads)
gaussian_refine_kernel(const RefineArgs a, const gf_refine_outputs o) {
    const long long ba = static_cast<long long>(blockIdx.x) * kRefineThreads + threadIdx.x;
    if (ba >= a.total) return;
    const gf_refine_desc &d = a.d;
    const int D = d.out_dim, opa = d.include_opa, S = d.semantic_dim, s0 = 10 + opa;
    const float *row = a.out + ba * D, *arow = a.anchor + ba * d.anchor_dim;
    const Frame f = refine_frame(a, row, arow);
    float *na = o.new_anchor + ba * D;
#pragma unroll
    for (int i = 0; i < 6; ++i) na[i] = __double2float_rn(f.o[i]);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        na[6 + i] = __double2float_rn(f.rot[i]);
        o.rotations[4 * ba + i] = __double2float_rn(f.rot[i]);
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        o.means[3 * ba + i] = __double2float_rn(f.sm[i].s * static_cast<double>(d.extent[i]) + static_cast<double>(d.lo[i]));
        o.scales[3 * ba + i] =
            __double2float_rn(static_cast<double>(d.scale_lo) + static_cast<double>(d.scale_extent) * f.ss[i].s);
        if (d.variant == GF_REFINE_V2) {
            o.original_means[3 * ba + i] = __double2float_rn(f.orig[i]);
            o.delta_means[3 * ba + i] = __double2float_rn(f.delta[i]);
        }
    }
    if (opa) {
        const double v = column(a, row, arow, 10);
        na[10] = __double2float_rn(v);
        o.opacities[ba] = __double2float_rn(safe_sigmoid(v).s);
    }
    float *sem = o.semantics + ba * S;
    if (d.semantics_act == GF_REFINE_SOFTMAX) {
        double x[kMaxSem], m = -INFINITY, sum = 0.0;
#pragma unroll
        for (int k = 0; k < kMaxSem; ++k)
            if (k < S) {
                x[k] = column(a, row, arow, s0 + k);
                na[s0 + k] = __double2float_rn(x[k]);
                m = fmax(m, x[k]);
            }
#pragma unroll
        for (int k = 0; k < kMaxSem; ++k)
            if (k < S) {
                x[k] = exp(x[k] - m);
                sum += x[k];
            }
#pragma unroll
        for (int k = 0; k < kMaxSem; ++k)
            if (k < S) sem[k] = __double2float_rn(x[k] / sum);
    } else {
        const bool softplus = d.semantics_act == GF_REFINE_SOFTPLUS;
        for (int k = 0; k < S; ++k) {
            const double v = column(a, row, arow, s0 + k);
            na[s0 + k] = __double2float_rn(v);
            sem[k] = __double2float_rn(softplus && v <= kSoftplusThreshold ? log1p(exp(v)) : v);
        }
    }
}

// one thread per (b, a).  dO[j] = d loss / d o[j] from the gradients of the outputs, then back through the
// normalisation, the residual add and the restriction (V1) or the inverse sigmoid and the two position maps (V2).
__global__ void __launch_bounds__(kRefineThreads)
gaussian_refine_grad_kernel(const RefineArgs a, const gf_refine_grads g, float *__restrict__ grad_out,
                            float *__restrict__ grad_anchor) {
    const long long ba = static_cast<long long>(blockIdx.x) * kRefineThreads + threadIdx.x;
    if (ba >= a.total) return;
    const gf_refine_desc &d = a.d;
    const int D = d.out_dim, Da = d.anchor_dim, opa = d.include_opa, S = d.semantic_dim, s0 = 10 + opa;
    const int r = d.refine_prefix;
    const float *row = a.out + ba * D, *arow = a.anchor + ba * Da;
    const Frame f = refine_frame(a, row, arow);
    float *go = grad_out + ba * D, *ga = grad_anchor + ba * Da;
    double dO[10];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        dO[i] = grad_at(g.new_anchor, ba * D + i) +
                grad_at(g.means, 3 * ba + i) * static_cast<double>(d.extent[i]) * f.sm[i].ds;
        dO[3 + i] = grad_at(g.new_anchor, ba * D + 3 + i) +
                    grad_at(g.scales, 3 * ba + i) * static_cast<double>(d.scale_extent) * f.ss[i].ds;
    }
    double gr[4], dot = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        gr[i] = grad_at(g.new_anchor, ba * D + 6 + i) + grad_at(g.rotations, 4 * ba + i);
        dot += f.rot[i] * gr[i];
    }
    if (f.below_eps) dot = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) dO[6 + i] = f.inv_norm * (gr[i] - f.rot[i] * dot);

    if (d.variant == GF_REFINE_V1) {
#pragma unroll
        for (int i = 0; i < 10; ++i) {
            const double gi = (i < 3 && d.restrict_xyz) ? dO[i] * 2.0 * static_cast<double>(d.unit[i]) * f.sr[i].ds
                                                        : dO[i];
            go[i] = __double2float_rn(gi);
            if (i < Da) ga[i] = i < r ? __double2float_rn(dO[i]) : 0.f;
        }
    } else {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const double ext = d.extent[i];
            const double dt = f.tin[i] ? dO[i] / (f.tc[i] * (1.0 - f.tc[i])) : 0.0;
            const double dsum = dt / ext;                              // d (orig + delta)
            const double dorig = dsum + grad_at(g.original_means, 3 * ba + i);
            const double ddelta = dsum + grad_at(g.delta_means, 3 * ba + i);
            ga[i] = __double2float_rn(dorig * ext * f.sa[i].ds);
            go[i] = __double2float_rn(ddelta * 2.0 * static_cast<double>(d.unit[i]) * f.sr[i].ds);
        }
#pragma unroll
        for (int i = 3; i < 10; ++i) {
            go[i] = __double2float_rn(dO[i]);
            if (i < Da) ga[i] = 0.f;
        }
    }

    // columns 10..D: the opacity and semantic logits, copied into new_anchor and activated
    auto emit = [&](int j, double v) {
        go[j] = __double2float_rn(v);
        if (j < Da) ga[j] = j < r ? __double2float_rn(v) : 0.f;
    };
    if (opa) {
        const double v = column(a, row, arow, 10);
        emit(10, grad_at(g.new_anchor, ba * D + 10) + grad_at(g.opacities, ba) * safe_sigmoid(v).ds);
    }
    const long long sem0 = ba * S;
    if (d.semantics_act == GF_REFINE_SOFTMAX) {
        double x[kMaxSem], m = -INFINITY, sum = 0.0, gdot = 0.0;
#pragma unroll
        for (int k = 0; k < kMaxSem; ++k)
            if (k < S) {
                x[k] = column(a, row, arow, s0 + k);
                m = fmax(m, x[k]);
            }
#pragma unroll
        for (int k = 0; k < kMaxSem; ++k)
            if (k < S) {
                x[k] = exp(x[k] - m);
                sum += x[k];
            }
#pragma unroll
        for (int k = 0; k < kMaxSem; ++k)
            if (k < S) {
                x[k] /= sum;                                           // the softmax y_k
                gdot += grad_at(g.semantics, sem0 + k) * x[k];
            }
#pragma unroll
        for (int k = 0; k < kMaxSem; ++k)
            if (k < S)
                emit(s0 + k, grad_at(g.new_anchor, ba * D + s0 + k) +
                                 (g.semantics != nullptr ? x[k] * (grad_at(g.semantics, sem0 + k) - gdot) : 0.0));
    } else {
        const bool softplus = d.semantics_act == GF_REFINE_SOFTPLUS;
        for (int k = 0; k < S; ++k) {
            double gs = grad_at(g.semantics, sem0 + k);
            if (softplus && g.semantics != nullptr) {
                const double v = column(a, row, arow, s0 + k);
                if (v <= kSoftplusThreshold) {
                    const double z = exp(v);
                    gs *= z / (z + 1.0);
                }
            }
            emit(s0 + k, grad_at(g.new_anchor, ba * D + s0 + k) + gs);
        }
    }
    for (int j = D; j < Da; ++j) ga[j] = 0.f;
}

// the checks both entry points share; *work = B * A (threads to launch)
static int check_refine(const gf_refine_desc *d, const float *out, const float *anchor, const char *what,
                        long long *work) {
    GF_REQUIRE(d != nullptr, GF_ERR_INVALID_ARG, "%s: desc is NULL", what);
    GF_REQUIRE(d->batch >= 0 && d->num_anchors >= 0 && d->out_dim >= 0 && d->anchor_dim >= 0 && d->semantic_dim >= 0 &&
                   d->refine_prefix >= 0,
               GF_ERR_INVALID_ARG, "%s: negative size (batch=%d, num_anchors=%d, out_dim=%d, anchor_dim=%d, "
               "semantic_dim=%d, refine_prefix=%d)", what, d->batch, d->num_anchors, d->out_dim, d->anchor_dim,
               d->semantic_dim, d->refine_prefix);
    GF_REQUIRE(d->variant == GF_REFINE_V1 || d->variant == GF_REFINE_V2, GF_ERR_INVALID_ARG, "%s: unknown variant %d",
               what, d->variant);
    GF_REQUIRE(d->semantics_act == GF_REFINE_IDENTITY || d->semantics_act == GF_REFINE_SOFTMAX ||
                   d->semantics_act == GF_REFINE_SOFTPLUS,
               GF_ERR_INVALID_ARG, "%s: unknown semantics activation %d", what, d->semantics_act);
    GF_REQUIRE((d->include_opa == 0 || d->include_opa == 1) && (d->restrict_xyz == 0 || d->restrict_xyz == 1),
               GF_ERR_INVALID_ARG, "%s: include_opa=%d and restrict_xyz=%d must be 0 or 1", what, d->include_opa,
               d->restrict_xyz);
    GF_REQUIRE(d->out_dim == 10 + d->include_opa + d->semantic_dim, GF_ERR_INVALID_ARG,
               "%s: out_dim=%d, expected 10 + include_opa + semantic_dim = %d", what, d->out_dim,
               10 + d->include_opa + d->semantic_dim);
    GF_REQUIRE(d->refine_prefix <= d->out_dim && d->refine_prefix <= d->anchor_dim, GF_ERR_INVALID_ARG,
               "%s: refine_prefix=%d exceeds min(out_dim=%d, anchor_dim=%d)", what, d->refine_prefix, d->out_dim,
               d->anchor_dim);
    if (d->variant == GF_REFINE_V2) {
        GF_REQUIRE(d->refine_prefix == 0 && d->restrict_xyz == 0, GF_ERR_INVALID_ARG,
                   "%s: refine_prefix and restrict_xyz are V1 fields and must be 0 for V2", what);
        GF_REQUIRE(d->anchor_dim >= 3, GF_ERR_INVALID_ARG, "%s: anchor_dim=%d, V2 reads the anchor's xyz logits",
                   what, d->anchor_dim);
    }
    GF_REQUIRE(d->semantic_dim <= GF_REFINE_MAX_SEMANTICS, GF_ERR_UNSUPPORTED,
               "%s: semantic_dim=%d is above the compiled maximum %d", what, d->semantic_dim, GF_REFINE_MAX_SEMANTICS);
    const long long ba = static_cast<long long>(d->batch) * d->num_anchors;
    const long long width = d->out_dim > d->anchor_dim ? d->out_dim : d->anchor_dim;
    GF_REQUIRE(ba < (1ll << 31) && ba * width < (1ll << 31), GF_ERR_UNSUPPORTED,
               "%s: batch * num_anchors * max(out_dim, anchor_dim) = %lld * %lld must stay below 2^31", what, ba,
               width);
    *work = ba;
    if (ba == 0) return GF_OK;
    GF_REQUIRE(out != nullptr, GF_ERR_INVALID_ARG, "%s: out is NULL", what);
    if (d->anchor_dim > 0) GF_REQUIRE(anchor != nullptr, GF_ERR_INVALID_ARG, "%s: anchor is NULL", what);
    return GF_OK;
}

static RefineArgs refine_args(const gf_refine_desc *d, long long total, const float *out, const float *anchor) {
    RefineArgs a;
    a.d = *d; a.total = total;
    a.out = out; a.anchor = anchor;
    return a;
}

static unsigned refine_blocks(long long total) {
    return static_cast<unsigned>((total + kRefineThreads - 1) / kRefineThreads);
}

}  // namespace gf

using namespace gf;

extern "C" {

int gf_gaussian_refine(const gf_refine_desc *desc, const float *out, const float *anchor,
                       const gf_refine_outputs *outputs, gf_stream_t stream_) {
    const char *what = "gaussian refine";
    long long total = 0;
    int rc = check_refine(desc, out, anchor, what, &total);
    if (rc != GF_OK) return rc;
    if (total == 0) return GF_OK;
    GF_REQUIRE(outputs != nullptr, GF_ERR_INVALID_ARG, "%s: outputs is NULL", what);
    const gf_refine_outputs &o = *outputs;
    GF_REQUIRE(o.new_anchor && o.means && o.scales && o.rotations, GF_ERR_INVALID_ARG,
               "%s: new_anchor, means, scales or rotations is NULL", what);
    if (desc->include_opa) GF_REQUIRE(o.opacities != nullptr, GF_ERR_INVALID_ARG, "%s: opacities is NULL", what);
    if (desc->semantic_dim > 0) GF_REQUIRE(o.semantics != nullptr, GF_ERR_INVALID_ARG, "%s: semantics is NULL", what);
    if (desc->variant == GF_REFINE_V2)
        GF_REQUIRE(o.original_means && o.delta_means, GF_ERR_INVALID_ARG,
                   "%s: original_means or delta_means is NULL", what);
    const RefineArgs a = refine_args(desc, total, out, anchor);
    gaussian_refine_kernel<<<refine_blocks(total), kRefineThreads, 0, static_cast<cudaStream_t>(stream_)>>>(a, o);
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}

int gf_gaussian_refine_backward(const gf_refine_desc *desc, const float *out, const float *anchor,
                                const gf_refine_grads *grads, float *grad_out, float *grad_anchor,
                                gf_stream_t stream_) {
    const char *what = "gaussian refine backward";
    long long total = 0;
    int rc = check_refine(desc, out, anchor, what, &total);
    if (rc != GF_OK) return rc;
    if (total == 0) return GF_OK;
    GF_REQUIRE(grad_out != nullptr, GF_ERR_INVALID_ARG, "%s: grad_out is NULL", what);
    if (desc->anchor_dim > 0) GF_REQUIRE(grad_anchor != nullptr, GF_ERR_INVALID_ARG, "%s: grad_anchor is NULL", what);
    gf_refine_grads g = {};
    if (grads != nullptr) g = *grads;
    const RefineArgs a = refine_args(desc, total, out, anchor);
    gaussian_refine_grad_kernel<<<refine_blocks(total), kRefineThreads, 0, static_cast<cudaStream_t>(stream_)>>>(
        a, g, grad_out, grad_anchor);
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}

}  // extern "C"
