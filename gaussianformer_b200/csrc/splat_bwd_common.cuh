// Shared pieces of the backward kernels (splat_backward.cu: one warp per Gaussian; splat_backward_bin.cu: one CTA per
// bin): launch parameters, per-pair arithmetic, the transposing warp reduction and the per-Gaussian epilogue.
#pragma once
#include "common.cuh"

namespace gf {

constexpr int kBigBox = 2048;
// CTA shapes of the two pair kernels: the prob variant carries more per-thread state, so it trades resident
// warps for registers (128 threads x 3 CTAs -> 168 registers) instead of spilling at 128.
constexpr int bwd_threads(bool prob) { return prob ? 128 : 256; }
constexpr int bwd_ctas(bool prob) { return prob ? 3 : 2; }

// Deterministic mode: the big kernel's grid per sample.  A constant, so that the (CTA, segment) split of the queue, and
// with it the summation order, depends on the inputs only (not on the SM count or the batch size).
constexpr int kDetBigCtas = 256;

// Launch parameters of every backward kernel: the call's desc and tensors, and the backward workspace.
//
// The workspace block is the one description of the workspace: only plan_backward_workspace (splat_backward.cu) sets
// it, kernels receive it whole and narrow it to one sample with sample_bwd.  Every pointer in it addresses B
// consecutive per-sample blocks, shaped as given; the deterministic-only regions (GF_BWD_DETERMINISTIC) are carved
// behind all others, so the layout without the flag is unchanged, and are NULL without it.
// The block stays flat and its first ten fields keep their offsets behind gr: the Gaussian-centric kernels run at
// their register cap, and ptxas allocates several of them differently (some with almost three times the spill
// traffic) when these fields move or sit in a struct of their own.  Check -Xptxas -v before reordering.
struct BwdParams {
    gf_splat_desc d;
    gf_splat_inputs in;
    gf_splat_grads gr;
    // ---- workspace
    int32_t *v2p;      // [H*W*D] per canon block: voxel -> largest point index in it, -1 for none
    uint2 *big;        // [B,G] queue of the boxes larger than kBigBox: (Gaussian, first chunk), ascending in both
    unsigned long long *big_ctr;   // [B] queue length << 40 | chunks queued (one atomic keeps the two in step)
    int chunk;         // box voxels per chunk, the unit of big and big_ctr
    // Per sample, cv_block bytes apart: the canon word (256 bytes, filled with 0xFF per call) directly in front of the
    // voxel -> point map, so that one memset covers all of them.  Non-zero after voxel_map_kernel iff N == H*W*D and
    // point n sits in voxel n for all n; word 1 is the route word (route_word).
    int32_t *canon;
    float4 *aux;       // [B,N] prob only: per-point terms that do not depend on the Gaussian
    size_t cv_block;   // bytes between the (canon, v2p) blocks of consecutive samples
    long long budget;  // deterministic: slot rows per sample
    uint32_t *det_cnt; // deterministic: [B,G] chunks of each Gaussian's box when it is queued for the big kernel, else 0
    float *det_part;   // deterministic: [B,G + kDetBigCtas,32] raw sums of the big kernel, one row per (CTA, entry) segment
    float *cov6;       // [B,G,6] gradient of Sigma^-1 when the caller passed scales + rotations instead of cov
    SplatWorkspace fwd;   // records, boxes and supertile lists for the bin-centric kernel
    float *sums;       // [B,32,G] raw sums of the bin-centric kernel (value-major), zero-filled by the host
    uint32_t *slot_off;   // deterministic: [B,G] first slot row of Gaussian g in the bin route
    float *slots;      // deterministic: [B,budget,32] raw sums of the bin route, one row per (Gaussian, bin) pair
    // ----
    int bin_active;    // the bin-centric kernel (splat_backward_bin.cu) serves this call when the points are canonical
};

// Word 1 of a sample's canon block (the 256 bytes in front of its voxel -> point map, filled with 0xFF per call): which
// route produced the gradients of a deterministic backward (GF_DEBUG_ROUTE_*, include/gf_b200_debug.h).
__host__ __device__ inline uint32_t *route_word(int32_t *canon) { return reinterpret_cast<uint32_t *>(canon) + 1; }
constexpr uint32_t kRouteBin = 0, kRouteSlotOverflow = 1, kRouteStrayPoints = 2, kRouteGaussian = 3;

// The launch parameters narrowed to sample b of the batch: its tensors and its blocks of the workspace.  The only code
// that computes per-sample offsets into the backward workspace.
__device__ __forceinline__ BwdParams sample_bwd(const BwdParams &p, int b) {
    BwdParams q = p;
    q.in = sample_inputs(p.d, p.in, b);
    q.gr = sample_grads(p.d, p.gr, b);
    q.canon = reinterpret_cast<int32_t *>(reinterpret_cast<char *>(p.canon) + b * p.cv_block);
    q.v2p = reinterpret_cast<int32_t *>(reinterpret_cast<char *>(p.v2p) + b * p.cv_block);
    q.big = p.big + static_cast<size_t>(b) * p.d.G;
    q.big_ctr = p.big_ctr + b;
    q.aux = adv(p.aux, static_cast<long long>(b) * p.d.N);
    q.cov6 = p.cov6 + static_cast<size_t>(b) * p.d.G * 6;
    q.fwd = sample_ws(p.fwd, p.d.G, b);
    q.sums = p.sums + static_cast<size_t>(b) * 32 * p.d.G;
    q.slot_off = adv(p.slot_off, static_cast<long long>(b) * p.d.G);
    q.slots = adv(p.slots, static_cast<long long>(b) * p.budget * 32);
    q.det_cnt = adv(p.det_cnt, static_cast<long long>(b) * p.d.G);
    q.det_part = adv(p.det_part, static_cast<long long>(b) * (p.d.G + kDetBigCtas) * 32);
    return q;
}

// Exclusive prefix sums of count(i), i = 0..n-1, in ascending i, by ONE CTA of NT threads: emit(i, prefix) for every
// i; returns the total.  Integer sums, so the result does not depend on timing.  Each pass covers NT * 8 values (eight
// consecutive ones per thread).
template <int NT, class Count, class Emit>
__device__ __forceinline__ unsigned long long cta_ordered_scan(int n, Count count, Emit emit) {
    constexpr int kPer = 8;
    __shared__ unsigned long long s_warp[NT / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned long long base = 0;
    for (int i0 = 0; i0 < n; i0 += NT * kPer) {
        unsigned long long v[kPer], sum = 0;
#pragma unroll
        for (int k = 0; k < kPer; ++k) {
            const int i = i0 + tid * kPer + k;
            v[k] = i < n ? count(i) : 0ull;
            sum += v[k];
        }
        unsigned long long incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        unsigned long long run = base + incl - sum, total = 0;
#pragma unroll
        for (int k = 0; k < NT / 32; ++k) {
            const unsigned long long c = s_warp[k];
            if (k < warp) run += c;
            total += c;
        }
        __syncthreads();   // s_warp is rewritten by the next pass
#pragma unroll
        for (int k = 0; k < kPer; ++k) {
            const int i = i0 + tid * kPer + k;
            if (i < n) emit(i, run);
            run += v[k];
        }
        base += total;
    }
    return base;
}

// One (Gaussian, point) pair's point-side data, fetched one iteration ahead of its use.
template <int C, bool PROB>
struct PairData {
    static constexpr int CP2 = (C + 1) / 2;
    static constexpr int kVec = (C + 2 + 3) / 4;   // float4 loads that cover a row starting 0 or 8 bytes into the first
    float px, py, pz;
    // dL/dlogits[n, :].  Wide mode (even C, 16-byte aligned base): the kVec aligned float4 that contain the
    // row, which starts at float `2*shift` of them -- a warp's 32 rows of 4C bytes then cost kVec
    // L1 passes instead of C/2.  Otherwise: packed pairs (zero padded for odd C) in raw[k/2].
    float4 raw[kVec];
    bool shift;
    float4 ax;                // prob: prob_aux_kernel's per-point terms
    bool ok;
    template <bool WIDE>
    __device__ __forceinline__ float2 up(int k) const {   // k is a compile-time constant after unrolling
        if (WIDE) {
            const float2 a = (k & 1) ? make_float2(raw[k >> 1].z, raw[k >> 1].w) : make_float2(raw[k >> 1].x, raw[k >> 1].y);
            const int k1 = k + 1;
            const float2 b = (k1 & 1) ? make_float2(raw[k1 >> 1].z, raw[k1 >> 1].w) : make_float2(raw[k1 >> 1].x, raw[k1 >> 1].y);
            return shift ? b : a;
        }
        return (k & 1) ? make_float2(raw[k >> 1].z, raw[k >> 1].w) : make_float2(raw[k >> 1].x, raw[k >> 1].y);
    }
};

// Per-Gaussian constants and running sums of one thread.  The sums are kept in the form that needs the
// fewest instructions per pair; the linear maps to the actual gradients are applied once per Gaussian
// (finish()):  d(mean) = -A * sum(w d),  d(cov) = -(1/2 | 1) * sum(w d d^T) (+ det terms for prob).
template <int C, bool PROB>
struct GaussAcc {
    static constexpr int CP2 = (C + 1) / 2;
    // constants
    float mu[3], q6[6];       // q6: exponent coefficients pre-scaled by log2(e)
    float opa, norm, inv2det; // prob: kappa*sqrt(det), 0.5/det
    float2 sem[CP2];
    // sums
    float sd[3];      // sum w * d
    float so;         // opacity gradient
    float2 ss[CP2];   // semantics gradient (base: without the common factor opa)
    float sq[6];      // sum w * (dx^2, dy^2, dz^2, dx dy, dy dz, dx dz)
    float sg;         // prob: sum of gamma

    __device__ __forceinline__ void load(const BwdParams &p, int g) {
#pragma unroll
        for (int a = 0; a < 3; ++a) mu[a] = p.in.means[3 * g + a];
        float c6[6];
        load_cov6_in(p.d, p.in, g, c6);
        q6[0] = -0.5f * kLog2e * c6[0]; q6[1] = -0.5f * kLog2e * c6[1]; q6[2] = -0.5f * kLog2e * c6[2];
        q6[3] = -kLog2e * c6[3]; q6[4] = -kLog2e * c6[4]; q6[5] = -kLog2e * c6[5];
        opa = p.in.opacities[g];
        if (PROB) {
            const float det = c6[0] * c6[1] * c6[2] + 2.f * c6[3] * c6[4] * c6[5] - c6[0] * c6[4] * c6[4] -
                              c6[1] * c6[5] * c6[5] - c6[2] * c6[3] * c6[3];
            norm = kKappa * sqrtf(det);
            inv2det = __fdiv_rn(0.5f, det);
        } else {
            norm = 0.f; inv2det = 0.f;
        }
#pragma unroll
        for (int k = 0; k < CP2; ++k) {
            sem[k].x = p.in.semantics[static_cast<size_t>(g) * C + 2 * k];
            sem[k].y = (2 * k + 1 < C) ? p.in.semantics[static_cast<size_t>(g) * C + 2 * k + 1] : 0.f;
            ss[k] = make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) sd[a] = 0.f;
        so = 0.f; sg = 0.f;
#pragma unroll
        for (int a = 0; a < 6; ++a) sq[a] = 0.f;
    }

    // the same constants from a raw record of the pack kernel (splat_prep.cu, PackParams.raw):
    // floats [0,3) mean, 3 opacity, [4,10) inverse covariance (xx,yy,zz,xy,yz,xz), [12,12+C) class vector
    __device__ __forceinline__ void load_record(const float4 *rec) {
        const float4 r0 = __ldg(rec), r1 = __ldg(rec + 1), r2 = __ldg(rec + 2);
        mu[0] = r0.x; mu[1] = r0.y; mu[2] = r0.z;
        opa = r0.w;
        const float c6[6] = {r1.x, r1.y, r1.z, r1.w, r2.x, r2.y};
        q6[0] = -0.5f * kLog2e * c6[0]; q6[1] = -0.5f * kLog2e * c6[1]; q6[2] = -0.5f * kLog2e * c6[2];
        q6[3] = -kLog2e * c6[3]; q6[4] = -kLog2e * c6[4]; q6[5] = -kLog2e * c6[5];
        if (PROB) {
            const float det = c6[0] * c6[1] * c6[2] + 2.f * c6[3] * c6[4] * c6[5] - c6[0] * c6[4] * c6[4] -
                              c6[1] * c6[5] * c6[5] - c6[2] * c6[3] * c6[3];
            norm = kKappa * sqrtf(det);
            inv2det = __fdiv_rn(0.5f, det);
        } else {
            norm = 0.f; inv2det = 0.f;
        }
#pragma unroll
        for (int q = 0; q < (C + 3) / 4; ++q) {
            const float4 v = __ldg(rec + 3 + q);
            sem[2 * q] = make_float2(v.x, v.y);
            if (2 * q + 1 < CP2) sem[2 * q + 1] = make_float2(v.z, v.w);
        }
        zero_sums();
    }
    __device__ __forceinline__ void zero_sums() {
#pragma unroll
        for (int k = 0; k < CP2; ++k) ss[k] = make_float2(0.f, 0.f);
#pragma unroll
        for (int a = 0; a < 3; ++a) sd[a] = 0.f;
        so = 0.f; sg = 0.f;
#pragma unroll
        for (int a = 0; a < 6; ++a) sq[a] = 0.f;
    }

    // issue the loads of point n (n < 0: no point in that voxel)
    template <bool WIDE>
    __device__ __forceinline__ void fetch(const BwdParams &p, long long n, PairData<C, PROB> &o) const {
        o.ok = n >= 0;
        if (!o.ok) return;
        o.px = __ldg(p.in.pts + 3 * n); o.py = __ldg(p.in.pts + 3 * n + 1); o.pz = __ldg(p.in.pts + 3 * n + 2);
        const float *row = p.gr.logits_grad + n * C;
        if (WIDE) {
            // 4C bytes starting 8-byte aligned: the enclosing 16-byte aligned window of kVec float4
            o.shift = (reinterpret_cast<uintptr_t>(row) & 8) != 0;
            const float4 *w = reinterpret_cast<const float4 *>(row - (o.shift ? 2 : 0));
#pragma unroll
            for (int k = 0; k < PairData<C, PROB>::kVec - 1; ++k) o.raw[k] = __ldg(w + k);
            constexpr int last = PairData<C, PROB>::kVec - 1;
            // the last float4 of an unshifted row may reach past the row; past the tensor for the last row
            if ((C % 4) == 2 && !o.shift && n + 1 >= p.d.N) {
                const float2 t = __ldg(reinterpret_cast<const float2 *>(w + last));
                o.raw[last] = make_float4(t.x, t.y, 0.f, 0.f);
            } else if ((C % 4) == 0 && !o.shift) {
                o.raw[last] = make_float4(0.f, 0.f, 0.f, 0.f);   // C % 4 == 0: the unshifted row ends with float4 last-1
            } else {
                o.raw[last] = __ldg(w + last);
            }
        } else if ((C & 1) == 0 && (reinterpret_cast<uintptr_t>(p.gr.logits_grad) & 7) == 0) {   // rows are 8-byte aligned
#pragma unroll
            for (int k = 0; k < CP2; ++k) {
                const float2 t = __ldg(reinterpret_cast<const float2 *>(row) + k);
                if (k & 1) { o.raw[k >> 1].z = t.x; o.raw[k >> 1].w = t.y; } else { o.raw[k >> 1].x = t.x; o.raw[k >> 1].y = t.y; }
            }
        } else {
#pragma unroll
            for (int k = 0; k < CP2; ++k) {
                const float a = __ldg(row + 2 * k);
                const float b = (2 * k + 1 < C) ? __ldg(row + 2 * k + 1) : 0.f;
                if (k & 1) { o.raw[k >> 1].z = a; o.raw[k >> 1].w = b; } else { o.raw[k >> 1].x = a; o.raw[k >> 1].y = b; }
            }
        }
        if (PROB) o.ax = __ldg(p.aux + n);
    }

    // contribution of one pair (the point lies inside the box)
    template <bool WIDE>
    __device__ __forceinline__ void consume(const PairData<C, PROB> &d) {
        if (!d.ok) return;
        const float dx = mu[0] - d.px, dy = mu[1] - d.py, dz = mu[2] - d.pz;
        float t1 = q6[0] * dx;
        t1 = fmaf(q6[3], dy, t1);
        t1 = fmaf(q6[5], dz, t1);
        float t2 = q6[1] * dy;
        t2 = fmaf(q6[4], dz, t2);
        float q = t1 * dx;
        q = fmaf(t2, dy, q);
        q = fmaf(q6[2] * dz, dz, q);
        const float E = ex2_approx(q);
        float w;  // weight of the geometric terms: d(loss)/d(power) * E
        if (!PROB) {
            // backward.cu:72-87 with t = sum_k sem_k * up_k
            float2 t = make_float2(0.f, 0.f);
            const float2 EE = make_float2(E, E);
#pragma unroll
            for (int k = 0; k < CP2; ++k) {
                const float2 u = d.template up<WIDE>(k);
                t = ffma2(sem[k], u, t);
                ss[k] = ffma2(u, EE, ss[k]);   // * opa at the end
            }
            const float et = E * (t.x + t.y);
            so += et;
            w = opa * et;
        } else {
            // localagg_prob/src/backward.cu:76-100 with the point-only terms pre-folded (prob_aux_kernel)
            const float Pt = norm * E;
            float pi = 0.f;
            if (d.ax.w > 0.f) {
                float2 u2 = make_float2(-d.ax.x, 0.f);
                const float sfac = Pt * opa * d.ax.w;
                const float2 ff = make_float2(sfac, sfac);
#pragma unroll
                for (int k = 0; k < CP2; ++k) {
                    const float2 uk = d.template up<WIDE>(k);
                    u2 = ffma2(uk, sem[k], u2);
                    ss[k] = ffma2(uk, ff, ss[k]);
                }
                const float u = u2.x + u2.y;
                pi = u * opa * d.ax.w;
                so = fmaf(u * Pt, d.ax.w, so);
            }
            const float eps = pi * norm + __fdividef(d.ax.y, 1.f - E + 1e-9f) + d.ax.z;
            sg = fmaf(pi * Pt, inv2det, sg);
            w = eps * E;
        }
        const float wx = w * dx, wy = w * dy, wz = w * dz;
        sd[0] += wx; sd[1] += wy; sd[2] += wz;
        sq[0] = fmaf(wx, dx, sq[0]);
        sq[1] = fmaf(wy, dy, sq[1]);
        sq[2] = fmaf(wz, dz, sq[2]);
        sq[3] = fmaf(wx, dy, sq[3]);
        sq[4] = fmaf(wy, dz, sq[4]);
        sq[5] = fmaf(wx, dz, sq[5]);
    }

    // The sums as a 32-vector in the order of the output lanes: [0,3) mean, 3 opacity, [4,10) cov,
    // [10,10+C) semantics, 10+C gamma (prob).  C <= 21.
    static constexpr int kVals = 10 + C + (PROB ? 1 : 0);
    static_assert(kVals <= 32, "one lane per reduced value");
    __device__ __forceinline__ void to_vector(float x[32]) const {
#pragma unroll
        for (int i = 0; i < 32; ++i) x[i] = 0.f;
#pragma unroll
        for (int a = 0; a < 3; ++a) x[a] = sd[a];
        x[3] = so;
#pragma unroll
        for (int a = 0; a < 6; ++a) x[4 + a] = sq[a];
#pragma unroll
        for (int k = 0; k < C; ++k) x[10 + k] = (k & 1) ? ss[k >> 1].y : ss[k >> 1].x;
        if (PROB) x[10 + C] = sg;
    }
};

// Sum of x[i] over the warp for all i at once: afterwards lane L holds the total of x[L] (in x[0]).
// 31 shuffles instead of 5 per value.
__device__ __forceinline__ float warp_transpose_reduce(float x[32], int lane) {
#pragma unroll
    for (int h = 16; h >= 1; h >>= 1) {
        const bool upper = (lane & h) != 0;
#pragma unroll
        for (int i = 0; i < h; ++i) {
            const float send = upper ? x[i] : x[i + h];
            const float keep = upper ? x[i + h] : x[i];
            x[i] = keep + __shfl_xor_sync(0xffffffffu, send, h);
        }
    }
    return x[0];
}

// Lane L holds the warp/CTA total of value L (see to_vector).  Applies the per-Gaussian linear maps and
// writes (or atomically adds) the gradients of Gaussian g.
template <int C, bool PROB>
__device__ __forceinline__ void finish(const BwdParams &p, int g, float v, int lane, bool atomic) {
    const float s0 = __shfl_sync(0xffffffffu, v, 0), s1 = __shfl_sync(0xffffffffu, v, 1), s2 = __shfl_sync(0xffffffffu, v, 2);
    const float sg = PROB ? __shfl_sync(0xffffffffu, v, 10 + C) : 0.f;
    float c6[6];
    load_cov6_in(p.d, p.in, g, c6);
    const float a = c6[0], b = c6[1], c = c6[2], d = c6[3], e = c6[4], f = c6[5];
    float out = 0.f;
    float *dst = nullptr;   // lane >= 10 + C: nothing to store
    if (lane < 3) {
        // -(A * sum w d): rows (a d f), (d b e), (f e c)
        const float r0 = lane == 0 ? a : (lane == 1 ? d : f);
        const float r1 = lane == 0 ? d : (lane == 1 ? b : e);
        const float r2 = lane == 0 ? f : (lane == 1 ? e : c);
        out = -(r0 * s0 + r1 * s1 + r2 * s2);
        dst = p.gr.means_grad + 3 * g + lane;
    } else if (lane == 3) {
        out = v;
        dst = p.gr.opacity_grad + g;
    } else if (lane < 10) {
        const int i = lane - 4;
        out = (i < 3) ? -0.5f * v : -v;
        if (PROB) {
            const float m[6] = {b * c - e * e, a * c - f * f, a * b - d * d,
                                2.f * (e * f - c * d), 2.f * (d * f - a * e), 2.f * (d * e - b * f)};
            float mi = m[0];
#pragma unroll
            for (int j = 1; j < 6; ++j) mi = (i == j) ? m[j] : mi;
            out = fmaf(sg, mi, out);
        }
        if (p.d.cov_stride == 9) {
            // gradient in the layout of the 3x3 input: the six gathered entries [0,4,8,1,5,2] receive it, the
            // lower triangle gets zero (what indexing autograd produces in the reference, __init__.py:143)
            const int flat = (i < 3) ? 4 * i : (i == 3 ? 1 : (i == 4 ? 5 : 2));
            dst = p.gr.cov_grad + 9 * static_cast<size_t>(g) + flat;
            if (!atomic && i < 3) p.gr.cov_grad[9 * static_cast<size_t>(g) + (i == 0 ? 3 : 5 + i)] = 0.f;
        } else {
            dst = p.gr.cov_grad + 6 * static_cast<size_t>(g) + i;
        }
    } else if (lane < 10 + C) {
        out = PROB ? v : p.in.opacities[g] * v;
        dst = p.gr.semantics_grad + static_cast<size_t>(g) * C + (lane - 10);
    }
    if (dst) {
        if (atomic) atomicAdd(dst, out); else *dst = out;
    }
}

// Walks the flat indices first, first+stride, ... < end of a box (z fastest) without a division per
// step: the stride is decomposed once into (sx, sy, sz) box steps and applied with two carries.
// Grid voxel indices fit 32 bits (H*W*D < 2^31 is checked at the C ABI).
struct BoxWalk {
    int nx, ny, nz;
    long long vol;
    int vbase;   // grid voxel index of the box corner
    int WD, D;
    int ix, iy, iz, sx, sy, sz;
    int left;    // steps this thread still has to take
    __device__ __forceinline__ void init(const int l[3], const int h[3], bool empty, int W, int D_) {
        nx = empty ? 0 : h[0] - l[0] + 1;
        ny = empty ? 0 : h[1] - l[1] + 1;
        nz = empty ? 0 : h[2] - l[2] + 1;
        vol = static_cast<long long>(nx) * ny * nz;
        D = D_; WD = W * D_;
        vbase = empty ? 0 : (l[0] * W + l[1]) * D_ + l[2];
    }
    __device__ __forceinline__ void start(long long first, long long end, int stride) {
        if (end > vol) end = vol;
        left = first < end ? static_cast<int>((end - first + stride - 1) / stride) : 0;
        if (left == 0) { ix = iy = iz = sx = sy = sz = 0; return; }
        iz = static_cast<int>(first % nz);
        const long long t = first / nz;
        iy = static_cast<int>(t % ny);
        ix = static_cast<int>(t / ny);
        sz = stride % nz;
        const int t2 = stride / nz;
        sy = t2 % ny;
        sx = t2 / ny;
    }
    __device__ __forceinline__ bool valid() const { return left > 0; }
    __device__ __forceinline__ int voxel() const { return vbase + ix * WD + iy * D + iz; }
    __device__ __forceinline__ void step() {
        --left;
        iz += sz;
        const int cz = iz >= nz;
        iz -= cz ? nz : 0;
        iy += sy + cz;
        const int cy = iy >= ny;
        iy -= cy ? ny : 0;
        ix += sx + cy;
    }
};


}  // namespace gf
