// Splat stage 1 — per-Gaussian packing and supertile binning (no host synchronisation, no sort).
//
// The reference builds a (voxel, Gaussian) pair list, radix-sorts it and needs a blocking D2H copy
// of the pair count in the middle (model/head/localagg/src/aggregator_impl.cu:193-230).  Here:
//
//   pack_mask_kernel   one thread per Gaussian: fuses the reference's Python host preparation
//                      (trunc voxel index of the mean, ceil radius, 3x3 -> 6 gather;
//                      local_aggregate/__init__.py:137-143) with FORWARD::preprocess
//                      (src/forward.cu:9-28): writes a 128-byte record (mean, exponent
//                      coefficients pre-scaled by log2(e), amplitude, class vector), the clipped
//                      integer box, and one ballot bit per supertile (16x16 columns) it overlaps.
//   list_kernel        one CTA per supertile: popcount-scan of the mask words -> ascending
//                      Gaussian index list (ascending order == the reference's stable sort order).
#include "splat_host.cuh"

namespace gf {

struct PackParams {
    gf_splat_desc d;
    gf_splat_inputs in;
    SplatWorkspace ws;
    int raw;     // != 0: records for the bin-centric backward -- (mu, opacity | c6 as given | sem as given), nothing folded
};

constexpr int kMaskPass = 1024;  // supertiles resolved per shared-memory pass

__global__ void __launch_bounds__(kPackThreads) pack_mask_kernel(const PackParams p) {
    __shared__ uint32_t s_mask[kPackThreads / 32][kMaskPass];
    __shared__ uint32_t s_err;
    const int g = blockIdx.x * kPackThreads + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool live = g < p.d.G;
    // sample b of the batch: its input tensors and its blocks of the workspace regions (the region sizes are the same
    // for every sample and are read from p.ws)
    const int b = blockIdx.y;
    const gf_splat_inputs in = sample_inputs(p.d, p.in, b);
    const SplatWorkspace ws = sample_ws(p.ws, p.d.G, b);
    if (threadIdx.x == 0) s_err = 0;
    pdl_launch_dependents();   // the list kernel may become resident now; it waits for this grid before reading

    uint32_t err = 0;
    int lo[3] = {1, 1, 1}, hi[3] = {0, 0, 0};
    bool empty = true;
    if (live) {
        // ---- every load first (read-only path), then arithmetic, then stores ------------------------
        const float mu[3] = {__ldg(in.means + 3 * g), __ldg(in.means + 3 * g + 1), __ldg(in.means + 3 * g + 2)};
        float c6[6];
        load_cov6_in(p.d, in, g, c6);   // the caller's Sigma^-1, or R^T diag(1/s^2) R from scales + rotations (cov == NULL)
        float amp = __ldg(in.opacities + g);
        const int nq = (p.ws.rec - kGeomFloats) / 4;   // <= 5 for C <= 20
        float semv[20];
        {
            const float *sem = in.semantics + static_cast<size_t>(g) * p.d.C;
#pragma unroll
            for (int i = 0; i < 20; ++i) semv[i] = (i < p.d.C) ? __ldg(sem + i) : 0.f;
        }
        empty = gaussian_box(p.d, in, g, mu, lo, hi, err);

        PackedBox bx;
        bx.x = empty ? 1u : (static_cast<uint32_t>(lo[0]) | static_cast<uint32_t>(hi[0]) << 16);
        bx.y = empty ? 1u : (static_cast<uint32_t>(lo[1]) | static_cast<uint32_t>(hi[1]) << 16);
        bx.z = empty ? 1u : (static_cast<uint32_t>(lo[2]) | static_cast<uint32_t>(hi[2]) << 16);
        bx.empty = empty ? 1u : 0u;
        ws.boxes[g] = bx;

        const float a_ = c6[0], b_ = c6[1], c_ = c6[2], d_ = c6[3], e_ = c6[4], f_ = c6[5];
        if (p.raw) {
            // backward: the kernel needs the opacity, the inverse covariance and the class vector themselves
        } else if (p.d.variant == GF_SPLAT_PROB) {
            // (2*pi)^-1.5 * sqrt(det) * opacity   (localagg_prob/src/forward.cu:77-78)
            const float det = a_ * b_ * c_ + 2.f * d_ * e_ * f_ - a_ * e_ * e_ - b_ * f_ * f_ - c_ * d_ * d_;
            amp = kKappa * sqrtf(det) * amp;
        } else {
            // base variant: out = sum_g (o_g s_g) E_g -- the opacity rides in the class vector, the render kernels
            // multiply by E alone (one multiply per Gaussian here instead of one per (voxel, Gaussian) pair there)
#pragma unroll
            for (int i = 0; i < 20; ++i) semv[i] *= amp;
            // ... which frees the amplitude slot: it carries the z levels the clipped box covers as a bit mask (grids of
            // up to 32 levels), so the tile kernel's column loop needs no list entry to know which of a lane's four
            // voxels lie inside the box (one shared load per step less)
            uint32_t zmask = 0u;
            if (!empty && p.d.D <= 32) zmask = ((2u << hi[2]) - 1u) & ~((1u << lo[2]) - 1u);
            amp = __uint_as_float(zmask);
        }
        float4 *rec = reinterpret_cast<float4 *>(ws.records + static_cast<size_t>(g) * p.ws.rec);
        rec[0] = make_float4(mu[0], mu[1], mu[2], amp);
        if (p.raw) {
            rec[1] = make_float4(a_, b_, c_, d_);
            rec[2] = make_float4(e_, f_, 0.f, 0.f);
#pragma unroll
            for (int q = 0; q < 5; ++q)
                if (q < nq) rec[3 + q] = make_float4(semv[4 * q], semv[4 * q + 1], semv[4 * q + 2], semv[4 * q + 3]);
        } else {   // forward layout (common.cuh): classes 16, 17 ride in the coefficient chunk
            rec[1] = make_float4(-0.5f * kLog2e * a_, -0.5f * kLog2e * b_, -0.5f * kLog2e * c_, -kLog2e * d_);
            rec[2] = make_float4(-kLog2e * e_, -kLog2e * f_, semv[16], semv[17]);
#pragma unroll
            for (int q = 0; q < 4; ++q) rec[3 + q] = make_float4(semv[4 * q], semv[4 * q + 1], semv[4 * q + 2], semv[4 * q + 3]);
            if (nq > 4) rec[7] = make_float4(semv[18], semv[19], 0.f, 0.f);
        }
    }

    // ---- supertile masks: per-warp words assembled in shared memory, stored by all lanes ------------
    const int sx0 = empty ? 1 : lo[0] / p.ws.st, sx1 = empty ? 0 : hi[0] / p.ws.st;
    const int sy0 = empty ? 1 : lo[1] / p.ws.st, sy1 = empty ? 0 : hi[1] / p.ws.st;
    const int word = g >> 5;          // warp-uniform
    const int nsuper = p.ws.nsuper;
    if (word < p.ws.nwords) {
        for (int base = 0; base < nsuper; base += kMaskPass) {
            const int npass = min(kMaskPass, nsuper - base);
            for (int i = lane; i < npass; i += 32) s_mask[warp][i] = 0u;
            __syncwarp();
            // a lane sets its own bits when its box touches few supertiles; a box that touches many (the
            // whole-grid "empty" Gaussian touches all of them) is spread over the 32 lanes instead
            const int ny = sy1 - sy0 + 1, cnt = empty ? 0 : (sx1 - sx0 + 1) * ny;
            const bool wide = cnt > 16;
            if (!wide)   // a column of each supertile the box touches
                for (int x = sx0 * p.ws.st; x <= sx1 * p.ws.st; x += p.ws.st)
                    for (int y = sy0 * p.ws.st; y <= sy1 * p.ws.st; y += p.ws.st) {
                        const int s = supertile_of(p.ws, x, y) - base;
                        if (s >= 0 && s < npass) atomicOr(&s_mask[warp][s], 1u << lane);
                    }
            uint32_t wides = __ballot_sync(0xffffffffu, wide);
            while (wides) {
                const int src = __ffs(wides) - 1;
                wides &= wides - 1;
                const int wx0 = __shfl_sync(0xffffffffu, sx0, src), wy0 = __shfl_sync(0xffffffffu, sy0, src);
                const int wny = __shfl_sync(0xffffffffu, ny, src), wcnt = __shfl_sync(0xffffffffu, cnt, src);
                for (int i = lane; i < wcnt; i += 32) {
                    const int s = supertile_of(p.ws, (wx0 + i / wny) * p.ws.st, (wy0 + i % wny) * p.ws.st) - base;
                    if (s >= 0 && s < npass) atomicOr(&s_mask[warp][s], 1u << src);
                }
            }
            __syncwarp();
            for (int i = lane; i < npass; i += 32)
                ws.masks[static_cast<size_t>(base + i) * p.ws.nwords + word] = s_mask[warp][i];
            __syncwarp();
        }
    }

    // ---- per-CTA error bits (plain store; list_kernel folds them into the status word) ----------
    __syncthreads();
    if (err) atomicOr(&s_err, err);
    __syncthreads();
    if (threadIdx.x == 0) p.ws.pack_flags[blockIdx.y * gridDim.x + blockIdx.x] = s_err;
}

struct ListParams {
    SplatWorkspace ws;
    int G;
    uint32_t initial_flags;
};

constexpr int kListThreads = 256;
constexpr int kListWordsPerThread = 4;   // consecutive mask words per thread and pass (keeps ascending order)

__global__ void __launch_bounds__(kListThreads) list_kernel(const ListParams p) {
    const SplatWorkspace ws = sample_ws(p.ws, p.G, blockIdx.y);
    const int s = blockIdx.x;   // supertile s of sample blockIdx.y
    const uint32_t *words = ws.masks + static_cast<size_t>(s) * ws.nwords;
    int32_t *list = ws.lists + static_cast<size_t>(s) * p.G;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __shared__ int s_warp[2][kListThreads / 32];
    pdl_launch_dependents();   // lets the render kernel start its point prologue
    pdl_wait();                // masks and flags of the pack kernel are complete from here on
    int base = 0, pass = 0;
    for (int w0 = 0; w0 < ws.nwords; w0 += kListThreads * kListWordsPerThread, ++pass) {
        const int first = w0 + threadIdx.x * kListWordsPerThread;
        uint32_t bits[kListWordsPerThread];
        int cnt = 0;
#pragma unroll
        for (int i = 0; i < kListWordsPerThread; ++i) {
            bits[i] = first + i < ws.nwords ? __ldg(words + first + i) : 0u;
            cnt += __popc(bits[i]);
        }
        int incl = cnt;  // inclusive warp scan
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) s_warp[pass & 1][warp] = incl;
        __syncthreads();
        int warp_off = 0, total = 0;
#pragma unroll
        for (int k = 0; k < kListThreads / 32; ++k) {
            const int c = s_warp[pass & 1][k];
            if (k < warp) warp_off += c;
            total += c;
        }
        int pos = base + warp_off + incl - cnt;
#pragma unroll
        for (int i = 0; i < kListWordsPerThread; ++i) {
            uint32_t b = bits[i];
            while (b) {
                const int bit = __ffs(b) - 1;
                b &= b - 1;
                list[pos++] = (first + i) * 32 + bit;
            }
        }
        base += total;
    }
    if (threadIdx.x == 0) ws.counts[s] = base;

    if (s == 0 && blockIdx.y == 0) {  // fold the pack kernel's error bits into the status word (also initialises it)
        uint32_t e = 0;
        for (int i = threadIdx.x; i < ws.pack_ctas * ws.batch; i += kListThreads) e |= ws.pack_flags[i];
        e = __reduce_or_sync(0xffffffffu, e);
        __shared__ uint32_t s_e;
        if (threadIdx.x == 0) s_e = p.initial_flags;
        __syncthreads();
        if (lane == 0 && e) atomicOr(&s_e, e);
        __syncthreads();
        if (threadIdx.x == 0) ws.flags[0] = s_e;
        else if (threadIdx.x < 32) ws.flags[threadIdx.x] = 0u;   // words 4..19: cycle counters of a GF_RENDER_TIMING build
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
SplatWorkspace plan_forward_workspace(const gf_splat_desc &d, WorkspaceCarver &carve) {
    SplatWorkspace ws;
    // supertile edge in columns: a power of two and a multiple of both render bin edges (8 and 4)
    int st = 16;
    const size_t budget = size_t(512) << 20;
    while (true) {
        const size_t ns = size_t((d.H + st - 1) / st) * size_t((d.W + st - 1) / st);
        if (ns * size_t(d.G) * 4 <= budget || st >= 1024) break;
        st *= 2;
    }
    ws.rec = rec_floats(d.C);
    ws.st = st;
    ws.nsx = (d.H + st - 1) / st;
    ws.nsy = (d.W + st - 1) / st;
    ws.nsuper = ws.nsx * ws.nsy;
    ws.nwords = (d.G + 31) / 32;
    ws.pack_ctas = (d.G + kPackThreads - 1) / kPackThreads;
    ws.batch = batch_of(d);
    const size_t B = static_cast<size_t>(ws.batch);
    ws.flags = carve.take<uint32_t>(256);
    ws.pack_flags = carve.take<uint32_t>(B * ws.pack_ctas * 4);
    ws.records = carve.take<float>(B * d.G * ws.rec * 4);
    ws.boxes = carve.take<PackedBox>(B * d.G * sizeof(PackedBox));
    ws.masks = carve.take<uint32_t>(B * ws.nsuper * ws.nwords * 4);
    ws.lists = carve.take<int32_t>(B * ws.nsuper * d.G * 4);
    ws.counts = carve.take<int32_t>(B * ws.nsuper * 4);
    return ws;
}

int launch_prep(const gf_splat_desc &d, const gf_splat_inputs &in, const SplatWorkspace &ws,
                uint32_t initial_flags, cudaStream_t stream, bool raw_records) {
    if (ws.pack_ctas > 0) {
        pack_mask_kernel<<<dim3(ws.pack_ctas, ws.batch), kPackThreads, 0, stream>>>(PackParams{d, in, ws, raw_records ? 1 : 0});
        GF_CUDA_TRY(cudaGetLastError());
    }
    GF_REQUIRE(ws.batch <= 65535, GF_ERR_UNSUPPORTED, "splat: batch above 65535");
    GF_CUDA_TRY(launch_chained(list_kernel, dim3(ws.nsuper, ws.batch), dim3(kListThreads), 0, stream, ListParams{ws, d.G, initial_flags}));
    return GF_OK;
}

}  // namespace gf
