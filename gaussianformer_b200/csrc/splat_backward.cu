// Splat backward (replaces BACKWARD::preprocess / BACKWARD::renderCUDA,
// model/head/localagg/src/backward.cu:8-20,24-103 and model/head/localagg_prob/src/backward.cu:24-123).
//
// The reference walks each Gaussian's box serially in ONE thread (640 000 iterations for the
// "empty" Gaussian of the solid config).  Here the walk is parallel and needs nothing saved by the
// forward pass:
//
//   voxel_map_kernel      voxel -> point index (largest index wins; the reference's write is a race)
//   backward_small_kernel one warp per Gaussian whose clipped box holds <= kBigBox voxels: lanes
//                         stride over the box (division-free walk, loads one pair ahead, packed
//                         fp32 pairs for the class sums), 28 (+1) partial sums in registers, one
//                         transposing warp reduction, plain stores (deterministic).  Larger boxes
//                         are queued.
//   backward_big_kernel   the queued boxes, measured in chunks of kBigChunk box voxels, form one long
//                         line of work; every CTA takes an equal contiguous span of it (balanced by
//                         volume: the whole-grid Gaussian is spread over the whole GPU, while a span
//                         of small queued boxes is walked Gaussian by Gaussian); block reduction +
//                         one atomicAdd per scalar and (CTA, Gaussian) segment.
#include "splat_bwd_common.cuh"
#include "splat_host.cuh"

namespace gf {

__global__ void __launch_bounds__(256) voxel_map_kernel(const BwdParams pb) {
    pdl_launch_dependents();   // the pair kernels may become resident; they wait before using the map
    const BwdParams p = sample_bwd(pb, blockIdx.y);
    if (p.bin_active) {   // launched behind the bin-centric kernel, which verified the point order: canonical -> done
        pdl_wait();
        if (*p.canon != 0) return;
    }
    const int H = p.d.H, W = p.d.W, D = p.d.D;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        *p.big_ctr = 0ull;
        if (static_cast<long long>(p.d.N) != static_cast<long long>(H) * W * D) *p.canon = 0;   // can only be generic
    }
    for (long long n = blockIdx.x * 256ll + threadIdx.x; n < p.d.N; n += 256ll * gridDim.x) {
        int ix, iy, iz;
        if (p.in.points_int) {
            ix = p.in.points_int[3 * n]; iy = p.in.points_int[3 * n + 1]; iz = p.in.points_int[3 * n + 2];
        } else {
            ix = voxel_coord(p.in.pts[3 * n], p.d.pc_min[0], p.d.grid_size);
            iy = voxel_coord(p.in.pts[3 * n + 1], p.d.pc_min[1], p.d.grid_size);
            iz = voxel_coord(p.in.pts[3 * n + 2], p.d.pc_min[2], p.d.grid_size);
        }
        if (ix < 0 || ix >= H || iy < 0 || iy >= W || iz < 0 || iz >= D) { *p.canon = 0; continue; }
        const long long v = (static_cast<long long>(ix) * W + iy) * D + iz;
        if (v != n) *p.canon = 0;   // benign race: every writer stores 0 (the memset left it non-zero)
        atomicMax(p.v2p + v, static_cast<int>(n));
    }
}

// Prob variant: everything in localagg_prob/src/backward.cu:76-100 that depends on the point only is
// folded into one float4 per point, read once per (Gaussian, point) pair instead of 2C+4 scalars:
//   x = sum_k dL/dlogits[n,k] * logits[n,k]     (so that sum_k up_k (sem_k - logits_k) = up.sem - x)
//   y = (1 - bin_logits[n]) * dL/dbin[n]
//   z = dL/ddensity[n]
//   w = 1 / probability[n]  if probability[n] > 1e-9 else 0   (0 switches the logits branch off)
__global__ void __launch_bounds__(256) prob_aux_kernel(const BwdParams pb, int C) {
    pdl_launch_dependents();
    const BwdParams p = sample_bwd(pb, blockIdx.y);
    for (long long n = blockIdx.x * 256ll + threadIdx.x; n < p.d.N; n += 256ll * gridDim.x) {
        float x = 0.f;
        for (int k = 0; k < C; ++k) x = fmaf(__ldg(p.gr.logits_grad + n * C + k), __ldg(p.gr.logits + n * C + k), x);
        const float Z = __ldg(p.gr.probability + n);
        p.aux[n] = make_float4(x, (1.f - __ldg(p.gr.bin_logits + n)) * __ldg(p.gr.bin_logits_grad + n),
                               __ldg(p.gr.density_grad + n), Z > 1e-9f ? __fdiv_rn(1.f, Z) : 0.f);
    }
    // runs beside voxel_map_kernel (nothing above depends on it) but must not COMPLETE before it: the pair
    // kernel's wait only covers the grid launched immediately before it
    pdl_wait();
}

// The pair loop of one thread, software pipelined by one iteration (the loads of pair i+1 are in
// flight while pair i is evaluated).
template <int C, bool PROB, bool WIDE>
__device__ __forceinline__ void walk_pairs_t(const BwdParams &p, GaussAcc<C, PROB> &acc, BoxWalk &box, bool canon) {
    PairData<C, PROB> pa, pb;
    auto next = [&](PairData<C, PROB> &o) -> bool {   // false: the walk is over
        if (!box.valid()) { o.ok = false; return false; }
        const int v = box.voxel();
        acc.template fetch<WIDE>(p, canon ? v : __ldg(p.v2p + v), o);
        box.step();
        return true;
    };
    bool more = next(pa);
    while (more) {
        more = next(pb);
        acc.template consume<WIDE>(pa);
        if (!more) { acc.template consume<WIDE>(pb); break; }
        more = next(pa);
        acc.template consume<WIDE>(pb);
        if (!more) acc.template consume<WIDE>(pa);
    }
}

template <int C, bool PROB>
__device__ __forceinline__ void walk_pairs(const BwdParams &p, GaussAcc<C, PROB> &acc, BoxWalk &box, bool canon) {
    // wide rows need an even class count and a 16-byte aligned gradient tensor (uniform for the launch)
    if ((C & 1) == 0 && (reinterpret_cast<uintptr_t>(p.gr.logits_grad) & 15) == 0)
        walk_pairs_t<C, PROB, true>(p, acc, box, canon);
    else
        walk_pairs_t<C, PROB, false>(p, acc, box, canon);
}

// DET (deterministic mode): a box above kBigBox is not enqueued with an atomic; its chunk count goes to det_cnt[g] (0 for
// the other boxes) and queue_scan_kernel builds the queue in ascending g.
template <int C, bool PROB, bool STRIDED, bool DET>
__device__ __forceinline__ void backward_small(const BwdParams &pb) {
    constexpr int kBwdThreads = bwd_threads(PROB);
    const BwdParams p = sample_bwd(pb, blockIdx.y);
    const int lane = threadIdx.x & 31;
    if (p.bin_active) {   // canonical points: the bin-centric kernel has produced the gradients; nothing to do here
        pdl_wait();
        if (*p.canon != 0) return;
    }
    // One Gaussian per warp and pass; the grid normally covers all Gaussians in one pass.  Behind the bin-centric kernel
    // this kernel is only its (rare) fallback and is launched with a small grid that strides over the Gaussians
    // (STRIDED; a separate instantiation, so that the one-pass kernel keeps its register allocation).
    const int per_cta = kBwdThreads / 32;
    const int passes = STRIDED ? (p.d.G + gridDim.x * per_cta - 1) / (gridDim.x * per_cta) : 1;
    bool waited = false;
#pragma unroll 1
    for (int pass = 0; pass < passes; ++pass) {
        // no early exit for the warps past G: they redo the last Gaussian and skip the stores, which keeps
        // every warp provably converged at the shuffles below
        const int g_raw = (pass * gridDim.x + blockIdx.x) * per_cta + (threadIdx.x >> 5);
        const bool live = g_raw < p.d.G;
        const int g = live ? g_raw : p.d.G - 1;
        GaussAcc<C, PROB> acc;
        acc.load(p, g);
        int lo[3], hi[3];
        uint32_t err = 0;
        const bool empty = gaussian_box(p.d, p.in, g, acc.mu, lo, hi, err) || !live;
        BoxWalk box;
        box.init(lo, hi, empty, p.d.W, p.d.D);
        const bool big = box.vol > kBigBox;
        if (!waited) {
            pdl_launch_dependents();
            pdl_wait();   // everything above read the caller's inputs only; the map, the canonical flag and the queue follow
            waited = true;
        }
        const bool canon = *p.canon != 0;   // then voxel index == point index and the map need not be read
        if (!big) {
            if (DET && lane == 0 && live) p.det_cnt[g] = 0u;
            box.start(lane, box.vol, 32);
            walk_pairs<C, PROB>(p, acc, box, canon);
        } else if (lane == 0) {   // (a big box is never the placeholder of a warp past G: that one is empty)
            const unsigned long long nch = static_cast<unsigned long long>((box.vol + p.chunk - 1) / p.chunk);
            if (DET) {
                p.det_cnt[g] = static_cast<uint32_t>(nch);
            } else {
                const unsigned long long old = atomicAdd(p.big_ctr, (1ull << 40) | nch);
                p.big[old >> 40] = make_uint2(static_cast<uint32_t>(g), static_cast<uint32_t>(old & ((1ull << 40) - 1)));
            }
        }
        // small boxes: final values; queued boxes: zeros (the big kernel accumulates atomically)
        float x[32];
        acc.to_vector(x);
        const float v = warp_transpose_reduce(x, lane);
        finish<C, PROB>(p, g, v, live ? lane : 32, false);
    }
}

template <int C, bool PROB, bool STRIDED>
__global__ void __launch_bounds__(bwd_threads(PROB), bwd_ctas(PROB)) backward_small_kernel(const BwdParams pb) {
    backward_small<C, PROB, STRIDED, false>(pb);
}

template <int C, bool PROB, bool STRIDED>
__global__ void __launch_bounds__(bwd_threads(PROB), bwd_ctas(PROB)) backward_small_det_kernel(const BwdParams pb) {
    backward_small<C, PROB, STRIDED, true>(pb);
}

// Deterministic mode: the big-box queue from backward_small_det_kernel's chunk counts, in ascending g (the order and
// chunk offsets the atomic enqueue would give if the warps arrived in Gaussian order).  One CTA per sample.
__global__ void __launch_bounds__(1024) queue_scan_kernel(const BwdParams pb) {
    pdl_launch_dependents();
    pdl_wait();
    const BwdParams p = sample_bwd(pb, blockIdx.x);
    if (threadIdx.x == 0 && !p.bin_active) *route_word(p.canon) = kRouteGaussian;
    if (p.bin_active && *p.canon != 0) return;
    const unsigned long long ctr = cta_ordered_scan<1024>(
        p.d.G,
        [&](int g) {
            const uint32_t c = p.det_cnt[g];
            return c ? (1ull << 40) | c : 0ull;
        },
        [&](int g, unsigned long long old) {
            if (p.det_cnt[g]) p.big[old >> 40] = make_uint2(static_cast<uint32_t>(g), static_cast<uint32_t>(old & ((1ull << 40) - 1)));
        });
    if (threadIdx.x == 0) *p.big_ctr = ctr;
}

// DET: every (CTA, queue entry) segment stores its raw sums to det_part row e + blockIdx.x (unique: a CTA's entries
// are consecutive and the next CTA starts at or after its last one) instead of adding finished gradients atomically;
// big_finish_kernel sums the rows of each entry.
template <int C, bool PROB, bool DET>
__device__ __forceinline__ void backward_big(const BwdParams &pb) {
    constexpr int kBwdThreads = bwd_threads(PROB);
    const BwdParams p = sample_bwd(pb, blockIdx.y);
    pdl_wait();
    if (p.bin_active && *p.canon != 0) return;   // (the queue is empty then anyway)
    const unsigned long long ctr = *p.big_ctr;
    const int nbig = static_cast<int>(ctr >> 40);
    const long long total = static_cast<long long>(ctr & ((1ull << 40) - 1));
    if (nbig == 0) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __shared__ float s_part[kBwdThreads / 32][32];
    const bool canon = *p.canon != 0;
    // my span of the chunk line, and the queue entry its first chunk belongs to (last entry with first <= lo)
    long long lo = total * blockIdx.x / gridDim.x;
    const long long hi = total * (blockIdx.x + 1) / gridDim.x;
    if (lo >= hi) return;
    int e = 0;
    for (int step = 1 << (31 - __clz(nbig)); step > 0; step >>= 1)
        if (e + step < nbig && static_cast<long long>(p.big[e + step].y) <= lo) e += step;
    for (; lo < hi; ++e) {
        const uint2 q = p.big[e];
        const int g = static_cast<int>(q.x);
        const long long next = (e + 1 < nbig) ? static_cast<long long>(p.big[e + 1].y) : total;
        const long long seg_end = next < hi ? next : hi;
        GaussAcc<C, PROB> acc;
        acc.load(p, g);
        int blo[3], bhi[3];
        uint32_t err = 0;
        const bool empty = gaussian_box(p.d, p.in, g, acc.mu, blo, bhi, err);
        BoxWalk box;
        box.init(blo, bhi, empty, p.d.W, p.d.D);
        const long long beg = (lo - q.y) * p.chunk;
        box.start(beg + threadIdx.x, (seg_end - q.y) * p.chunk, kBwdThreads);
        walk_pairs<C, PROB>(p, acc, box, canon);
        float x[32];
        acc.to_vector(x);
        const float v = warp_transpose_reduce(x, lane);
        s_part[warp][lane] = v;
        __syncthreads();
        if (warp == 0) {
            float tot = 0.f;
#pragma unroll
            for (int w = 0; w < kBwdThreads / 32; ++w) tot += s_part[w][lane];
            if (DET) p.det_part[static_cast<size_t>(e + blockIdx.x) * 32 + lane] = tot;
            else finish<C, PROB>(p, g, tot, lane, true);
        }
        __syncthreads();
        lo = seg_end;
    }
}

template <int C, bool PROB>
__global__ void __launch_bounds__(bwd_threads(PROB), bwd_ctas(PROB)) backward_big_kernel(const BwdParams pb) {
    backward_big<C, PROB, false>(pb);
}

template <int C, bool PROB>
__global__ void __launch_bounds__(bwd_threads(PROB), bwd_ctas(PROB)) backward_big_det_kernel(const BwdParams pb) {
    backward_big<C, PROB, true>(pb);
}

// DET: one warp per queue entry e.  The CTAs of backward_big_det_kernel whose chunk span meets the entry's chunks are
// k(first) .. k(last) with k(c) = ((c + 1) * kDetBigCtas - 1) / total (CTA k spans [total*k/grid, total*(k+1)/grid));
// those with an empty span wrote nothing.  Their rows are summed in ascending k and finish() writes the gradients,
// overwriting the zeros backward_small_det_kernel stored for the queued box.
template <int C, bool PROB>
__global__ void __launch_bounds__(256) big_finish_kernel(const BwdParams pb) {
    pdl_launch_dependents();
    pdl_wait();
    const BwdParams p = sample_bwd(pb, blockIdx.y);
    if (p.bin_active && *p.canon != 0) return;
    const unsigned long long ctr = *p.big_ctr;
    const int nbig = static_cast<int>(ctr >> 40);
    const long long total = static_cast<long long>(ctr & ((1ull << 40) - 1));
    const int e = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (e >= nbig) return;
    const uint2 q = p.big[e];
    const long long first = q.y, last = ((e + 1 < nbig) ? static_cast<long long>(p.big[e + 1].y) : total) - 1;
    const long long grid = kDetBigCtas;
    const long long k0 = ((first + 1) * grid - 1) / total, k1 = ((last + 1) * grid - 1) / total;
    float v = 0.f;
    for (long long k = k0; k <= k1; ++k)
        if (total * k / grid < total * (k + 1) / grid) v += p.det_part[static_cast<size_t>(e + k) * 32 + lane];
    finish<C, PROB>(p, static_cast<int>(q.x), v, lane, false);
}

// Gradients of the fused pre-op (in.cov == NULL): the [G,6] gradient of Sigma^-1 = R^T diag(1/s^2) R mapped to the
// scales and the (un-normalised) quaternion.  With U the upper-triangular matrix of the six gradients (only the six
// gathered entries of the 3x3 carry gradient, __init__.py:143) and Gs = U + U^T:
//   dL/dD_k = 1/2 r_k^T Gs r_k (r_k = row k of R),  dL/ds_k = -2/s_k^3 dL/dD_k,  dL/dR_kl = D_k (Gs r_k)_l,
// then through the quaternion -> matrix map (model/utils/utils.py:20-66) and F.normalize.
__global__ void __launch_bounds__(128) srt_grad_kernel(const BwdParams pb) {
    pdl_wait();
    const BwdParams p = sample_bwd(pb, blockIdx.y);
    const int g = blockIdx.x * 128 + threadIdx.x;
    if (g >= p.d.G) return;
    const float *g6 = p.gr.cov_grad + 6 * static_cast<size_t>(g);
    const float s[3] = {p.in.scales[3 * g], p.in.scales[3 * g + 1], p.in.scales[3 * g + 2]};
    const float q[4] = {p.in.rotations[4 * g], p.in.rotations[4 * g + 1], p.in.rotations[4 * g + 2], p.in.rotations[4 * g + 3]};
    float R[3][3], inv_norm;
    quat_rotation(q, R, inv_norm);
    const float Gs[3][3] = {{2.f * g6[0], g6[3], g6[5]}, {g6[3], 2.f * g6[1], g6[4]}, {g6[5], g6[4], 2.f * g6[2]}};
    float M[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float Dk = __fdiv_rn(1.f, s[k] * s[k]);
        float t[3];
#pragma unroll
        for (int l = 0; l < 3; ++l) t[l] = Gs[l][0] * R[k][0] + Gs[l][1] * R[k][1] + Gs[l][2] * R[k][2];
        const float dD = 0.5f * (R[k][0] * t[0] + R[k][1] * t[1] + R[k][2] * t[2]);
        p.gr.scales_grad[3 * g + k] = -2.f * dD * __fdiv_rn(Dk, s[k]);
#pragma unroll
        for (int l = 0; l < 3; ++l) M[k][l] = Dk * t[l];
    }
    // every quaternion takes the tangent projection here, as it always has: the splat's rotations are never near 0
    float dq[4];
    quat_rotation_backward(q, inv_norm, M, dq, false);
#pragma unroll
    for (int i = 0; i < 4; ++i) p.gr.rotations_grad[4 * g + i] = dq[i];
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// Byte counts of the backward workspace that only the host needs.
struct BwdPlan {
    size_t cv_bytes;     // the (canon word, voxel -> point map) blocks of all samples: one memset
    size_t sums_bytes;   // BwdParams::sums: one memset
    size_t bytes;        // the whole workspace
};

// Box voxels per chunk of the big-box kernel: 4 passes of a 256-thread CTA, grown when needed so that
// the chunk line of the worst case (every Gaussian covers the whole grid) stays below 2^31 chunks.
static int chunk_voxels(const gf_splat_desc &d) {
    const long long vox = static_cast<long long>(d.H) * d.W * d.D;
    long long c = 1024;
    while ((vox + c - 1) / c * static_cast<long long>(d.G > 0 ? d.G : 1) >= (1ll << 31)) c *= 2;
    return static_cast<int>(c);
}

// Slots per sample of the deterministic bin route (DESIGN.md 4.3).  The query sees the desc only, not the scales, so the
// budget is a formula of it: the base variant's boxes cover about 5 bins per Gaussian on the shipped configs, plus the
// whole-grid Gaussian's nbins_total; the prob variants' larger boxes up to about 50 bins per Gaussian.  A sample whose
// boxes need more slots is served by the Gaussian-centric chain instead.
static long long slot_budget(const gf_splat_desc &d) {
    const long long forced = slot_budget_override();
    if (forced >= 0) return forced;
    const long long nbins = static_cast<long long>((d.H + kBinX - 1) / kBinX) * ((d.W + kBinY - 1) / kBinY) * ((d.D + kBinZ - 1) / kBinZ);
    const long long b = d.variant == GF_SPLAT_PROB ? 64ll * d.G + nbins : 4ll * d.G + (1ll << 17) + nbins;
    return b < 0xffffffffll ? b : 0xffffffffll;   // slot numbers are 32-bit
}

// Carves the workspace at `base` (nullptr: only sizes it) into the workspace fields of ws.
BwdPlan plan_backward_workspace(const gf_splat_desc &d, uint32_t flags, void *base, BwdParams &ws) {
    WorkspaceCarver carve{static_cast<char *>(base)};
    const size_t B = static_cast<size_t>(batch_of(d));
    BwdPlan plan;
    ws.big_ctr = carve.take<unsigned long long>(B * 8);
    ws.cv_block = 256 + WorkspaceCarver::align(size_t(d.H) * d.W * d.D * 4);
    plan.cv_bytes = B * ws.cv_block;
    ws.canon = carve.take<int32_t>(plan.cv_bytes);
    ws.v2p = ws.canon ? ws.canon + 64 : nullptr;
    ws.big = carve.take<uint2>(B * size_t(d.G) * sizeof(uint2));
    ws.chunk = chunk_voxels(d);
    ws.aux = carve.take<float4>(d.variant == GF_SPLAT_PROB ? B * size_t(d.N) * 16 : 0);
    ws.cov6 = carve.take<float>(B * size_t(d.G) * 6 * 4);   // only used with scales + rotations input
    ws.fwd = plan_forward_workspace(d, carve);
    plan.sums_bytes = B * size_t(d.G) * 32 * 4;
    ws.sums = carve.take<float>(plan.sums_bytes);
    const bool det = (flags & GF_BWD_DETERMINISTIC) != 0;
    ws.budget = det ? slot_budget(d) : 0;
    ws.slot_off = det ? carve.take<uint32_t>(B * size_t(d.G) * 4) : nullptr;
    ws.slots = det ? carve.take<float>(B * size_t(ws.budget) * 32 * 4) : nullptr;
    ws.det_cnt = det ? carve.take<uint32_t>(B * size_t(d.G) * 4) : nullptr;
    ws.det_part = det ? carve.take<float>(B * (size_t(d.G) + kDetBigCtas) * 32 * 4) : nullptr;
    plan.bytes = carve.bytes;
    return plan;
}

size_t backward_workspace_bytes(const gf_splat_desc &d, uint32_t flags) {
    BwdParams ws{};
    return plan_backward_workspace(d, flags, nullptr, ws).bytes;
}

uint32_t *backward_route_words(const gf_splat_desc &d, void *workspace, size_t *stride) {
    BwdParams ws{};
    plan_backward_workspace(d, 0u, workspace, ws);
    *stride = ws.cv_block;
    return route_word(ws.canon);
}

template <int C, bool PROB>
static int launch_backward_t(const BwdParams &bp, const BwdPlan &plan, bool srt, bool det, int num_sms, cudaStream_t stream) {
    const gf_splat_desc &d = bp.d;
    const int B = batch_of(d);
    GF_REQUIRE(B <= 65535, GF_ERR_UNSUPPORTED, "splat backward: batch above 65535");
    // canon words (non-zero = "still canonical") and the voxel->point maps (-1 = empty) in one fill
    GF_CUDA_TRY(cudaMemsetAsync(bp.canon, 0xFF, plan.cv_bytes, stream));
    const long long want = (static_cast<long long>(d.N) + 255) / 256;
    const int grid0 = static_cast<int>(want < 16ll * num_sms ? (want > 0 ? want : 1) : 16ll * num_sms);
    if (bp.bin_active) {
        // Canonical points (checked by the bin kernel itself): memset -> [prob_aux] -> pack -> list -> bin -> finish, and
        // the Gaussian-centric chain below finds the flag set and returns.  pack is launched in plain stream order (it
        // starts when everything above has completed); the kernels after it are chained to their predecessor.
        // Deterministic mode: list -> slot plan -> bin (slot stores) -> slot reduce + finish; no accumulator to clear.
        if (!det) GF_CUDA_TRY(cudaMemsetAsync(bp.sums, 0, plan.sums_bytes, stream));   // accumulated with atomics
        if (PROB) {
            prob_aux_kernel<<<dim3(grid0, B), 256, 0, stream>>>(bp, C);
            GF_CUDA_TRY(cudaGetLastError());
        }
        int rc = launch_prep(d, bp.in, bp.fwd, 0u, stream, true);
        if (rc != GF_OK) return rc;
        rc = launch_backward_bin(bp, det, stream);
        if (rc != GF_OK) return rc;
        // the Gaussian-centric chain is only the fallback now: small grids (they return at once when the points are canonical)
        GF_CUDA_TRY(launch_chained(voxel_map_kernel, dim3(num_sms, B), dim3(256), 0, stream, bp));
    } else {
        voxel_map_kernel<<<dim3(grid0, B), 256, 0, stream>>>(bp);   // plain stream order: never overlaps the previous call
        GF_CUDA_TRY(cudaGetLastError());
        if (PROB) GF_CUDA_TRY(launch_chained(prob_aux_kernel, dim3(grid0, B), dim3(256), 0, stream, bp, C));
    }
    constexpr int kBwdThreads = bwd_threads(PROB);
    const int per_cta = kBwdThreads / 32;
    int small_ctas = (d.G + per_cta - 1) / per_cta;
    int big_ctas = (num_sms * bwd_ctas(PROB) * 2 + B - 1) / B;   // per sample: together they fill the GPU twice over
    if (big_ctas < 32) big_ctas = 32;
    if (bp.bin_active) {
        if (small_ctas > num_sms) small_ctas = num_sms;
        big_ctas = num_sms;
    }
    if (det) {
        // the same chain with the queue built in Gaussian order, a constant big grid and an ordered sum of its segments
        if (bp.bin_active) GF_CUDA_TRY(launch_chained(backward_small_det_kernel<C, PROB, true>, dim3(small_ctas, B), dim3(kBwdThreads), 0, stream, bp));
        else GF_CUDA_TRY(launch_chained(backward_small_det_kernel<C, PROB, false>, dim3(small_ctas, B), dim3(kBwdThreads), 0, stream, bp));
        GF_CUDA_TRY(launch_chained(queue_scan_kernel, dim3(B), dim3(1024), 0, stream, bp));
        GF_CUDA_TRY(launch_chained(backward_big_det_kernel<C, PROB>, dim3(kDetBigCtas, B), dim3(kBwdThreads), 0, stream, bp));
        GF_CUDA_TRY(launch_chained(big_finish_kernel<C, PROB>, dim3((d.G + 7) / 8, B), dim3(256), 0, stream, bp));
    } else {
        if (bp.bin_active) GF_CUDA_TRY(launch_chained(backward_small_kernel<C, PROB, true>, dim3(small_ctas, B), dim3(kBwdThreads), 0, stream, bp));
        else GF_CUDA_TRY(launch_chained(backward_small_kernel<C, PROB, false>, dim3(small_ctas, B), dim3(kBwdThreads), 0, stream, bp));
        GF_CUDA_TRY(launch_chained(backward_big_kernel<C, PROB>, dim3(big_ctas, B), dim3(kBwdThreads), 0, stream, bp));
    }
    if (srt) GF_CUDA_TRY(launch_chained(srt_grad_kernel, dim3((d.G + 127) / 128, B), dim3(128), 0, stream, bp));
    return GF_OK;
}

int launch_backward(const gf_splat_desc &d, const gf_splat_inputs &in, const gf_splat_grads &gr, void *workspace,
                    uint32_t flags, int num_sms, cudaStream_t stream) {
    BwdParams bp{};
    bp.d = d;
    bp.in = in;
    bp.gr = gr;
    const BwdPlan plan = plan_backward_workspace(d, flags, workspace, bp);
    const bool srt = in.cov == nullptr;
    if (srt) {   // the pair kernels write the [G,6] gradient of Sigma^-1 into the workspace; srt_grad_kernel maps it on
        bp.d.cov_stride = 6;
        bp.gr.cov_grad = bp.cov6;
    }
    bp.bin_active = backward_bin_eligible(bp.d, bp.in, bp.gr) ? 1 : 0;
    const bool det = (flags & GF_BWD_DETERMINISTIC) != 0;
    const bool prob = d.variant == GF_SPLAT_PROB;
    return dispatch_classes(d.C, "splat backward", [&](auto cc) {
        constexpr int C = decltype(cc)::value;
        return prob ? launch_backward_t<C, true>(bp, plan, srt, det, num_sms, stream)
                    : launch_backward_t<C, false>(bp, plan, srt, det, num_sms, stream);
    });
}

}  // namespace gf
