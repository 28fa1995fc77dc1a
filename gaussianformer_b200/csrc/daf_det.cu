// Feature gradient of the deterministic deformable-aggregation backwards (GF_BWD_DETERMINISTIC).  The default route
// scatters it with vector atomics into feature rows that many points share, so its bits depend on the order the
// atomics land in.  Here the scatter is turned into a gather whose summation order is fixed by the inputs alone:
//
//   1. compact  one warp per sampling point emits its visible (camera, level) pairs in ascending pair id
//               bp*M*L + m*L + l; the positions come from an integer scan over the per-point counts
//   2. key      a pair's key is its top-left bilinear cell (b, m, l, y0, x0).  The gate 0 < loc < 1 puts y0 in
//               [-1, h-1] and x0 in [-1, w-1], so level l owns an extended (h+1) x (w+1) block of cells; the row
//               and column -1 are real (a point with y_im in (-0.5, 0) feeds its bottom corners only)
//   3. sort     stable LSD radix sort of the (key, pair id) entries over the key bits in use: per-tile digit
//               histograms, an exclusive scan, a stable in-tile scatter.  A cell's entries stay in ascending pair id
//   4. gather   one warp per feature row (b, m, level, y, x), lanes across the channels: the row is corner 0 of
//               cell (y, x), corner 1 of (y, x-1), corner 2 of (y-1, x) and corner 3 of (y-1, x-1); the cells are
//               visited in that order, each in ascending pair id, the coefficient of every entry is recomputed from
//               loc and the weights, and the fp32 sum is added (+=) to grad_feat once
//
// Every buffer is sized for the worst case (every pair visible) from the desc alone, and the visible count stays on
// the device: no host synchronisation, so the backward can be captured in a CUDA graph.
#include <algorithm>

#include "daf_pair.cuh"
#include "radix_sort.cuh"

namespace gf {
namespace {

constexpr size_t kAlign = 256;

// The workspace of the route, from the desc alone.  Cells: level l of (b, m) starts at sum_{k<l} (h_k+1)(w_k+1) of
// the (b, m) block, and the blocks are 2F + 2L cells apart, an upper bound of that sum for any level shapes with
// sum h_k w_k = F (h + w <= hw + 1 for h, w >= 1).
struct DetPlan {
    long long npairs, npts, ncells, cells_per_bm;
    int tiles, passes;
    size_t counts, partials, keys[2], vals[2], hist, cell_start, cell_end, bytes;
};

int det_plan(const gf_daf_desc &d, DetPlan &pl) {
    pl.npts = static_cast<long long>(d.batch) * d.num_pts;
    pl.npairs = pl.npts * d.num_cams * d.num_scale;
    pl.cells_per_bm = 2ll * d.num_feat + 2ll * d.num_scale;
    pl.ncells = static_cast<long long>(d.batch) * d.num_cams * pl.cells_per_bm;
    GF_REQUIRE(pl.npairs < (1ll << 31), GF_ERR_UNSUPPORTED,
               "daf deterministic backward: B*P*M*L = %lld (camera, level) pairs, the route takes fewer than 2^31",
               pl.npairs);
    GF_REQUIRE(pl.ncells < (1ll << 31), GF_ERR_UNSUPPORTED,
               "daf deterministic backward: B*M*(2F + 2L) = %lld cells, the route takes fewer than 2^31", pl.ncells);
    pl.tiles = static_cast<int>((pl.npairs + kSortTile - 1) / kSortTile);
    int bits = 0;
    while ((1ll << bits) < pl.ncells) ++bits;
    pl.passes = (bits + kRadixBits - 1) / kRadixBits;
    const long long scan_max = std::max(pl.npts + 1, static_cast<long long>(kRadix) * pl.tiles);
    size_t off = 0;
    auto take = [&](long long count, size_t elem) {
        const size_t at = off;
        off += (static_cast<size_t>(count) * elem + kAlign - 1) / kAlign * kAlign;
        return at;
    };
    pl.counts = take(pl.npts + 1, sizeof(int));   // per point, then its exclusive scan; the last entry is the total
    pl.partials = take((scan_max + kScanTile - 1) / kScanTile, sizeof(int));
    for (int i = 0; i < 2; ++i) {
        pl.keys[i] = take(pl.npairs, sizeof(uint32_t));
        pl.vals[i] = take(pl.npairs, sizeof(int));
    }
    pl.hist = take(static_cast<long long>(kRadix) * pl.tiles, sizeof(int));
    pl.cell_start = take(pl.ncells, sizeof(int));
    pl.cell_end = take(pl.ncells, sizeof(int));
    pl.bytes = off;
    return GF_OK;
}

struct DetParams {
    gf_daf_desc d;
    int K;                      // key points per anchor: the fused op's grad_out rows and stats are per anchor
    int cells_per_bm;
    long long ncells;
    int tiles;
    const int32_t *shape, *start;
    const float *loc;
    const uint8_t *pmask;       // fused: [B, A, K, M] or NULL
    const float *weights;       // plain: weights [B, P, M, L, Gr]; fused: logits of the same shape
    const uint8_t *wmask;       // fused: [B, A, K, M, L, Gr] or NULL
    const float *stats;         // fused: [B, A, Gr, 2] (max * log2e, 1 / sum); NULL for the plain op
    const float *grad_out;      // plain [B, P, C], fused [B, A, C]
    float *grad_feat;           // [B, M, F, C], +=
    int *counts;                // [B*P + 1]; counts[B*P] is the number of visible pairs after the scan
    int *partials;
    uint32_t *keys[2];
    int *vals[2];
    int *hist;                  // [kRadix, tiles]: digit-major, so one exclusive scan gives every (digit, tile) its start
    int *cell_start, *cell_end; // [ncells]: entry range of a cell in the sorted order (0, 0 = empty)
};

// ---------------------------------------------------------------------------------------------------------- compact
// Level table plus the first cell of every level inside a (b, m) block (le); every thread of the block must call it.
__device__ __forceinline__ void load_det_levels(const DetParams &p, int *lh, int *lw, int *ls, int *le) {
    load_level_table(p.d, p.shape, p.start, lh, lw, ls);
    if (threadIdx.x == 0) {
        int e = 0;
        for (int l = 0; l < p.d.num_scale; ++l) {
            le[l] = e;
            e += (lh[l] + 1) * (lw[l] + 1);
        }
    }
    __syncthreads();
}

// camera m sees point bp (cam_gate) and, fused, the point mask lets it through
__device__ __forceinline__ bool pair_visible(const DetParams &p, long long bp, int m, float &lx, float &ly) {
    return cam_gate(p.loc, bp, p.d.num_cams, m, lx, ly) && (!p.pmask || p.pmask[bp * p.d.num_cams + m] != 0);
}

__global__ void __launch_bounds__(kDafThreads) det_count_kernel(const DetParams p) {
    const int lane = threadIdx.x & 31;
    const int L = p.d.num_scale, npair = p.d.num_cams * L;
    const long long npts = static_cast<long long>(p.d.batch) * p.d.num_pts;
    const long long warps = static_cast<long long>(gridDim.x) * (kDafThreads / 32);
    for (long long bp = static_cast<long long>(blockIdx.x) * (kDafThreads / 32) + (threadIdx.x >> 5); bp < npts; bp += warps) {
        int cnt = 0;
        for (int pr0 = 0; pr0 < npair; pr0 += 32) {
            const int pr = pr0 + lane;
            float lx, ly;
            const bool vis = pr < npair && pair_visible(p, bp, pr / L, lx, ly);
            cnt += __popc(__ballot_sync(0xffffffffu, vis));
        }
        if (lane == 0) p.counts[bp] = cnt;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) p.counts[npts] = 0;
}

__global__ void __launch_bounds__(kDafThreads) det_emit_kernel(const DetParams p) {
    __shared__ int lh[kMaxLevels], lw[kMaxLevels], ls[kMaxLevels], le[kMaxLevels];
    load_det_levels(p, lh, lw, ls, le);
    const int lane = threadIdx.x & 31;
    const int M = p.d.num_cams, L = p.d.num_scale, npair = M * L;
    const long long npts = static_cast<long long>(p.d.batch) * p.d.num_pts;
    const long long warps = static_cast<long long>(gridDim.x) * (kDafThreads / 32);
    for (long long bp = static_cast<long long>(blockIdx.x) * (kDafThreads / 32) + (threadIdx.x >> 5); bp < npts; bp += warps) {
        const long long b = bp / p.d.num_pts;
        int pos = p.counts[bp];
        for (int pr0 = 0; pr0 < npair; pr0 += 32) {
            const int pr = pr0 + lane, m = pr / L, l = pr - m * L;
            float lx = 0.f, ly = 0.f;
            const bool vis = pr < npair && pair_visible(p, bp, m, lx, ly);
            const uint32_t ballot = __ballot_sync(0xffffffffu, vis);
            if (vis) {
                const int h = lh[l], w = lw[l];
                const BilinearCell cell = bilinear_cell(lx, ly, h, w);   // the cell whose corners pair_setup reads
                const long long key = (b * M + m) * p.cells_per_bm + le[l] + (cell.y0 + 1) * (w + 1) + (cell.x0 + 1);
                const int at = pos + __popc(ballot & lanemask_lt());
                p.keys[0][at] = static_cast<uint32_t>(key);
                p.vals[0][at] = static_cast<int>(bp * npair + pr);
            }
            pos += __popc(ballot);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------- sort
__global__ void __launch_bounds__(kSortThreads) radix_hist_kernel(const DetParams p, const uint32_t *keys, int shift) {
    const auto count = [&] { return static_cast<long long>(p.counts[static_cast<long long>(p.d.batch) * p.d.num_pts]); };
    radix_tile_hist(keys, count, shift, p.hist, p.tiles, blockIdx.x);
}

__global__ void __launch_bounds__(kSortThreads) radix_scatter_kernel(const DetParams p, const uint32_t *keys_in,
                                                                     const int *vals_in, uint32_t *keys_out,
                                                                     int *vals_out, int shift) {
    const auto count = [&] { return static_cast<long long>(p.counts[static_cast<long long>(p.d.batch) * p.d.num_pts]); };
    radix_tile_scatter(keys_in, vals_in, keys_out, vals_out, count, shift, p.hist, p.tiles, blockIdx.x);
}

__global__ void __launch_bounds__(256) cell_bounds_kernel(const DetParams p, const uint32_t *keys) {
    const long long n = p.counts[static_cast<long long>(p.d.batch) * p.d.num_pts];
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t k = keys[i];
        if (k >= p.ncells) continue;   // a level table whose sizes do not add up to num_feat
        if (i == 0 || keys[i - 1] != k) p.cell_start[k] = static_cast<int>(i);
        if (i == n - 1 || keys[i + 1] != k) p.cell_end[k] = static_cast<int>(i + 1);
    }
}

// ---------------------------------------------------------------------------------------------------------- gather
// The aggregation weight of pair (bp, pr) for group grp: the plain op's weight, or the fused op's softmax_weight
template <bool FUSED>
__device__ __forceinline__ float pair_weight(const DetParams &p, long long bp, int pr, int grp, int npair) {
    const int Gr = p.d.num_groups;
    const long long widx = (bp * npair + pr) * Gr + grp;
    if (!FUSED) return __ldg(p.weights + widx);
    const float2 st = __ldg(reinterpret_cast<const float2 *>(p.stats + ((bp / p.K) * Gr + grp) * 2));
    return softmax_weight(__ldg(p.weights + widx), st.x, st.y, p.wmask, widx);
}

// Adds the entries [i_beg, i_end) of one cell, whose corner k is the warp's row, to this lane's channel slice c0 (4
// channels with VEC4, else 1 in acc.x), in entry order.  (h, w): the level's size; pr: the row's (camera, level) pair.
// The whole warp calls it; lanes past the last channel (active = false) only take part in the shuffles.
template <bool FUSED, bool VEC4>
__device__ __forceinline__ void gather_cell(const DetParams &p, const int *vals, int k, int i_beg, int i_end, int pr,
                                            int h, int w, int c0, int grp, bool active, float4 &acc) {
    const int lane = threadIdx.x & 31, C = p.d.num_embeds, M = p.d.num_cams, L = p.d.num_scale, npair = M * L;
    for (int i0 = i_beg; i0 < i_end; i0 += 32) {
        // lane e sets up entry i0 + e: its point and the bilinear weight of corner k of its cell (as in pair_setup)
        long long bp = 0;
        float cw = 0.f;
        if (i0 + lane < i_end) {
            bp = __ldg(vals + i0 + lane) / npair;
            const float *lp = p.loc + (bp * M + pr / L) * 2;
            cw = bilinear_cell(__ldg(lp), __ldg(lp + 1), h, w).weight(k);
        }
        const int nb = min(32, i_end - i0);
        for (int e = 0; e < nb; ++e) {
            const long long bpe = __shfl_sync(0xffffffffu, bp, e);
            const float cwe = __shfl_sync(0xffffffffu, cw, e);
            if (!active) continue;
            const float a = cwe * pair_weight<FUSED>(p, bpe, pr, grp, npair);
            const float *go = p.grad_out + (FUSED ? bpe / p.K : bpe) * C + c0;
            if (VEC4) {
                const float4 g = __ldg(reinterpret_cast<const float4 *>(go));
                acc.x += a * g.x; acc.y += a * g.y; acc.z += a * g.z; acc.w += a * g.w;
            } else {
                acc.x += a * __ldg(go);
            }
        }
    }
}

template <bool FUSED, bool VEC4>
__global__ void __launch_bounds__(kDafThreads) det_gather_kernel(const DetParams p, const int *vals) {
    __shared__ int lh[kMaxLevels], lw[kMaxLevels], ls[kMaxLevels], le[kMaxLevels];
    load_det_levels(p, lh, lw, ls, le);
    const int lane = threadIdx.x & 31;
    const int C = p.d.num_embeds, M = p.d.num_cams, L = p.d.num_scale, F = p.d.num_feat;
    const int gdim = C / p.d.num_groups;
    const long long rows = static_cast<long long>(p.d.batch) * M * F;
    const long long warps = static_cast<long long>(gridDim.x) * (kDafThreads / 32);
    for (long long r = static_cast<long long>(blockIdx.x) * (kDafThreads / 32) + (threadIdx.x >> 5); r < rows; r += warps) {
        const long long bm = r / F;
        const int f = static_cast<int>(r - bm * F);
        int l = 0;
        while (l < L && !(f >= ls[l] && f < ls[l] + lh[l] * lw[l])) ++l;
        if (l == L) continue;   // a row no level covers
        const int h = lh[l], w = lw[l];
        const int y = (f - ls[l]) / w, x = f - ls[l] - y * w;
        const int pr = static_cast<int>(bm % M) * L + l;
        int beg[4], end[4], any = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            // corner k of the cell (y - k/2, x - k%2) is this row
            const long long cell = bm * p.cells_per_bm + le[l] + (y - (k >> 1) + 1) * (w + 1) + (x - (k & 1) + 1);
            beg[k] = __ldg(p.cell_start + cell);
            end[k] = __ldg(p.cell_end + cell);
            any |= end[k] - beg[k];
        }
        if (any == 0) continue;
        constexpr int kSlice = VEC4 ? 128 : 32;   // channels per warp pass
        for (int s0 = 0; s0 < C; s0 += kSlice) {
            const int c0 = s0 + (VEC4 ? lane * 4 : lane);
            const bool active = c0 < C;
            const int grp = active ? c0 / gdim : 0;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            gather_cell<FUSED, VEC4>(p, vals, 0, beg[0], end[0], pr, h, w, c0, grp, active, acc);
            gather_cell<FUSED, VEC4>(p, vals, 1, beg[1], end[1], pr, h, w, c0, grp, active, acc);
            gather_cell<FUSED, VEC4>(p, vals, 2, beg[2], end[2], pr, h, w, c0, grp, active, acc);
            gather_cell<FUSED, VEC4>(p, vals, 3, beg[3], end[3], pr, h, w, c0, grp, active, acc);
            if (!active) continue;
            float *gf = p.grad_feat + r * C + c0;
            if (VEC4) {
                float4 v = *reinterpret_cast<float4 *>(gf);
                v.x += acc.x; v.y += acc.y; v.z += acc.z; v.w += acc.w;
                *reinterpret_cast<float4 *>(gf) = v;
            } else {
                *gf += acc.x;
            }
        }
    }
}

}  // namespace

size_t daf_det_workspace_bytes(const gf_daf_desc &d) {
    DetPlan pl;
    return det_plan(d, pl) == GF_OK ? pl.bytes : 0;
}

int launch_daf_det_feat_grad(const DafParams *p, const DafFusedParams *fp, void *workspace, int num_sms,
                             cudaStream_t stream) {
    DetParams q{};
    if (p) {
        q.d = p->d; q.K = 1; q.shape = p->shape; q.start = p->start; q.loc = p->loc; q.weights = p->weights;
        q.grad_out = p->grad_out; q.grad_feat = p->grad_feat;
    } else {
        q.d = fp->d; q.K = fp->K; q.shape = fp->shape; q.start = fp->start; q.loc = fp->loc; q.pmask = fp->pmask;
        q.weights = fp->logits; q.wmask = fp->wmask; q.stats = fp->stats; q.grad_out = fp->grad_out;
        q.grad_feat = fp->grad_feat;
    }
    DetPlan pl;
    const int rc = det_plan(q.d, pl);
    if (rc != GF_OK) return rc;
    if (pl.npts == 0) return GF_OK;
    char *ws = static_cast<char *>(workspace);
    q.cells_per_bm = static_cast<int>(pl.cells_per_bm);
    q.ncells = pl.ncells;
    q.tiles = pl.tiles;
    q.counts = reinterpret_cast<int *>(ws + pl.counts);
    q.partials = reinterpret_cast<int *>(ws + pl.partials);
    for (int i = 0; i < 2; ++i) {
        q.keys[i] = reinterpret_cast<uint32_t *>(ws + pl.keys[i]);
        q.vals[i] = reinterpret_cast<int *>(ws + pl.vals[i]);
    }
    q.hist = reinterpret_cast<int *>(ws + pl.hist);
    q.cell_start = reinterpret_cast<int *>(ws + pl.cell_start);
    q.cell_end = reinterpret_cast<int *>(ws + pl.cell_end);

    GF_CUDA_TRY(cudaMemsetAsync(q.cell_start, 0, pl.ncells * sizeof(int), stream));
    GF_CUDA_TRY(cudaMemsetAsync(q.cell_end, 0, pl.ncells * sizeof(int), stream));
    const int pt_grid = daf_grid(pl.npts, num_sms);
    det_count_kernel<<<pt_grid, kDafThreads, 0, stream>>>(q);
    int e = exclusive_scan(q.counts, pl.npts + 1, q.partials, stream);
    if (e != GF_OK) return e;
    det_emit_kernel<<<pt_grid, kDafThreads, 0, stream>>>(q);
    int cur = 0;
    for (int pass = 0; pass < pl.passes; ++pass, cur ^= 1) {
        radix_hist_kernel<<<pl.tiles, kSortThreads, 0, stream>>>(q, q.keys[cur], pass * kRadixBits);
        e = exclusive_scan(q.hist, static_cast<long long>(kRadix) * pl.tiles, q.partials, stream);
        if (e != GF_OK) return e;
        radix_scatter_kernel<<<pl.tiles, kSortThreads, 0, stream>>>(q, q.keys[cur], q.vals[cur], q.keys[cur ^ 1],
                                                                    q.vals[cur ^ 1], pass * kRadixBits);
    }
    cell_bounds_kernel<<<num_sms * 8, 256, 0, stream>>>(q, q.keys[cur]);
    const int row_grid = daf_grid(static_cast<long long>(q.d.batch) * q.d.num_cams * q.d.num_feat, num_sms);
    const bool v4 = q.d.num_embeds % 4 == 0 && (q.d.num_embeds / q.d.num_groups) % 4 == 0;
    if (fp) {
        det_gather_kernel<true, true><<<row_grid, kDafThreads, 0, stream>>>(q, q.vals[cur]);
    } else if (v4) {
        det_gather_kernel<false, true><<<row_grid, kDafThreads, 0, stream>>>(q, q.vals[cur]);
    } else {
        det_gather_kernel<false, false><<<row_grid, kDafThreads, 0, stream>>>(q, q.vals[cur]);
    }
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}

}  // namespace gf
