// Occupancy loss of one supervised layer (gf_occ_loss): OccupancyLoss.loss_voxel (loss/occupancy_loss.py:102-149) as
// the shipped configs run it -- weighted cross-entropy plus Lovasz-softmax (loss/utils/lovasz_softmax.py:157-234) --
// with its gradient, without a host synchronisation.  The voxels of the pool S (mask, b-major, n ascending) and the
// Lovasz set V (S without lovasz_ignore) are found on the device; every count stays there:
//
//   1. select   per voxel: S and V membership, the status bit of a label outside [0, C), |S| and the per-class
//               foreground counts of V (integer atomics); vpos[i] = voxel i is in V
//   2. scan     exclusive integer scan of vpos: a voxel's position in V, |V| in vpos[B*N]
//   3. keys     per voxel, fp64 inside: the CE term w[y] * -log p_y (block partials), and for every present class c
//               the error e = |[y = c] - r_c| rounded to fp32 once, stored as the key ~bits(e) at [c][position]
//   4. sort     one class-segmented stable LSD radix sort (radix_sort.cuh) of all classes at once: four 8-bit passes
//               over a [class][digit][tile] histogram; absent classes and tiles past |V| do no work.  Ascending
//               ~bits(e) is descending e, and equal errors keep ascending position in V
//   5. lovasz   per class in sorted order: an integer scan of the foreground, Delta_k = J_k - J_{k-1} in fp64, block
//               partials of e_k Delta_k, and dL_c/dr scattered to [c][position] through the sort's permutation
//               (a permutation per class: no atomics)
//   6. finish   one block: the partials summed in a fixed order, the loss and the two gradient scales
//   7. grad     per voxel: the softmax Jacobian (logits) or the identity (probabilities) applied to the Lovasz
//               gradient, plus the CE term, written in pred's layout, zeros included
//
// The workspace and every grid are sized from the desc for the worst case |V| = B*N, so loss and gradient are
// bit-reproducible from call to call and the op can be captured in a CUDA graph.
#include <algorithm>

#include "gf_b200_debug.h"
#include "radix_sort.cuh"

namespace gf {
namespace {

constexpr int kOccThreads = 256;
constexpr size_t kOccAlign = 256;
constexpr float kProbLo = 1e-6f, kProbHi = 1.f - 1e-6f;   // CE_wo_softmax's clamp as an fp32 tensor holds it
constexpr uint32_t kNegBit = 0x80000000u;                  // sort value: position in V | (fg - r < 0) << 31

struct OccHead {
    uint32_t status;          // GF_FLAG_LABEL_OUT_OF_RANGE
    int num_s;                // |S|
    double ce_scale;          // weight * ce_weight / sum_S w[y]
    double lov_scale;         // weight * lovasz_weight / (present classes), 0 when none is present
};

// Workspace of one call, from the desc alone.  pair[i] holds keys [C][B*N] uint32 then values [C][B*N] int; after
// the sort pair[1] is free and holds dL_c/dr as [C][B*N] doubles.
struct OccPlan {
    long long nvox, cv;
    int tiles, vox_blocks;
    size_t head, fg, vpos, partials, vlab, pair[2], hist, fgpart, lpart, cepart, bytes;
};

int occ_plan(const gf_occ_loss_desc &d, OccPlan &pl) {
    pl.nvox = static_cast<long long>(d.batch) * d.N;
    pl.cv = pl.nvox * d.C;
    GF_REQUIRE(pl.cv < (1ll << 31), GF_ERR_UNSUPPORTED,
               "occ loss: B*N*C = %lld (voxel, class) entries, the op takes fewer than 2^31", pl.cv);
    pl.tiles = static_cast<int>(std::max(1ll, (pl.nvox + kSortTile - 1) / kSortTile));
    pl.vox_blocks = static_cast<int>(std::max(1ll, (pl.nvox + kOccThreads - 1) / kOccThreads));
    const long long hist = static_cast<long long>(kRadix) * pl.tiles * d.C;
    size_t off = 0;
    auto take = [&](long long count, size_t elem) {
        const size_t at = off;
        off += (static_cast<size_t>(count) * elem + kOccAlign - 1) / kOccAlign * kOccAlign;
        return at;
    };
    pl.head = take(1, sizeof(OccHead));
    pl.fg = take(d.C, sizeof(int));                 // foreground count of every class in V
    pl.vpos = take(pl.nvox + 1, sizeof(int));
    pl.partials = take(scan_partials_count(std::max(pl.nvox + 1, hist)), sizeof(int));
    pl.vlab = take(pl.nvox, sizeof(uint8_t));       // label of every position in V (255: no class)
    for (int i = 0; i < 2; ++i) pl.pair[i] = take(2 * pl.cv, sizeof(uint32_t));
    pl.hist = take(hist, sizeof(int));
    pl.fgpart = take(static_cast<long long>(d.C) * pl.tiles, sizeof(int));
    pl.lpart = take(static_cast<long long>(d.C) * pl.tiles, sizeof(double));
    pl.cepart = take(2ll * pl.vox_blocks, sizeof(double));
    pl.bytes = off;
    return GF_OK;
}

struct OccParams {
    gf_occ_loss_desc d;
    long long nvox;
    int tiles;
    long long sb, sc, sn;     // element strides of pred / grad over (b, c, n)
    const float *pred;
    const int64_t *labels;
    const uint8_t *mask;
    const float *w;
    float *loss, *grad;
    OccHead *head;
    int *fg, *vpos, *fgpart;
    uint8_t *vlab;
    uint32_t *keys[2];
    int *vals[2];
    int *hist;
    double *dr;               // [C][B*N]: dL_c/dr at each position of V (aliases pair[1])
    double *lpart, *cepart;
};

struct Voxel {
    long long y;
    bool in_s, in_v;
};

__device__ __forceinline__ Voxel classify(const OccParams &p, long long i) {
    Voxel v;
    v.y = p.labels[i];
    v.in_s = !p.mask || p.mask[i] != 0;
    if (p.d.empty_label >= 0 && v.y == p.d.empty_label) v.in_s = false;
    v.in_v = v.in_s && v.y != p.d.lovasz_ignore;
    return v;
}

__device__ __forceinline__ bool has_class(const OccParams &p, long long y) { return y >= 0 && y < p.d.C; }

// fixed-order sum over the block of kOccThreads threads (shuffle tree, then the warps in order); valid in thread 0
__device__ __forceinline__ double block_sum(double v) {
    __shared__ double s[kOccThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kOccThreads / 32; ++w) t += s[w];
    return t;
}

// ---------------------------------------------------------------------------------------------------------- select
__global__ void __launch_bounds__(kOccThreads) occ_select_kernel(const OccParams p) {
    __shared__ int cnt[kMaxClasses];
    for (int c = threadIdx.x; c < p.d.C; c += kOccThreads) cnt[c] = 0;
    __syncthreads();
    const long long i = static_cast<long long>(blockIdx.x) * kOccThreads + threadIdx.x;
    bool in_s = false;
    if (i < p.nvox) {
        const Voxel v = classify(p, i);
        in_s = v.in_s;
        if (v.in_s && !has_class(p, v.y) && v.y != p.d.ignore_index && v.y != p.d.lovasz_ignore)
            atomicOr(&p.head->status, GF_FLAG_LABEL_OUT_OF_RANGE);
        if (v.in_v && has_class(p, v.y)) atomicAdd(&cnt[v.y], 1);
        p.vpos[i] = v.in_v ? 1 : 0;
    }
    if (i == 0) p.vpos[p.nvox] = 0;
    const int ns = __syncthreads_count(in_s);
    if (threadIdx.x == 0 && ns > 0) atomicAdd(&p.head->num_s, ns);
    for (int c = threadIdx.x; c < p.d.C; c += kOccThreads)
        if (cnt[c] > 0) atomicAdd(p.fg + c, cnt[c]);
}

// ---------------------------------------------------------------------------------------------------------- keys
template <int C, bool PROBS>
__global__ void __launch_bounds__(kOccThreads) occ_keys_kernel(const OccParams p) {
    const long long i = static_cast<long long>(blockIdx.x) * kOccThreads + threadIdx.x;
    double ce_num = 0.0, ce_den = 0.0;
    if (i < p.nvox) {
        const Voxel v = classify(p, i);
        if (v.in_s) {
            const long long b = i / p.d.N, n = i - b * p.d.N;
            const float *x = p.pred + b * p.sb + n * p.sn;
            double r[C];
#pragma unroll
            for (int c = 0; c < C; ++c) r[c] = __ldg(x + c * p.sc);
            double lse = 0.0;
            if (!PROBS) {   // r becomes the fp64 softmax
                double m = r[0];
#pragma unroll
                for (int c = 1; c < C; ++c) m = fmax(m, r[c]);
                double s = 0.0;
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    r[c] = exp(r[c] - m);
                    s += r[c];
                }
                lse = m + log(s);
#pragma unroll
                for (int c = 0; c < C; ++c) r[c] /= s;
            }
            if (has_class(p, v.y) && v.y != p.d.ignore_index) {
                const int y = static_cast<int>(v.y);
                const double wy = __ldg(p.w + y);
                double xy = 0.0;
#pragma unroll
                for (int c = 0; c < C; ++c) xy = c == y ? r[c] : xy;
                const double nll = PROBS ? -log(static_cast<double>(fminf(fmaxf(static_cast<float>(xy), kProbLo), kProbHi)))
                                         : lse - static_cast<double>(__ldg(x + y * p.sc));
                ce_num = wy * nll;
                ce_den = wy;
            }
            if (v.in_v) {
                const int at = p.vpos[i];
                p.vlab[at] = has_class(p, v.y) ? static_cast<uint8_t>(v.y) : uint8_t{255};
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    if (__ldg(p.fg + c) == 0) continue;   // absent class: never sorted
                    const double diff = (v.y == c ? 1.0 : 0.0) - r[c];
                    const float e = __double2float_rn(fabs(diff));
                    const long long k = c * p.nvox + at;
                    p.keys[0][k] = ~__float_as_uint(e);
                    p.vals[0][k] = at | (diff < 0.0 ? static_cast<int>(kNegBit) : 0);
                }
            }
        }
    }
    const double num = block_sum(ce_num), den = block_sum(ce_den);
    if (threadIdx.x == 0) {
        p.cepart[2 * blockIdx.x] = num;
        p.cepart[2 * blockIdx.x + 1] = den;
    }
}

// ---------------------------------------------------------------------------------------------------------- sort
// |V| for a present class, 0 for an absent one
__device__ __forceinline__ long long class_count(const OccParams &p, int c) {
    return p.fg[c] > 0 ? static_cast<long long>(p.vpos[p.nvox]) : 0ll;
}

// grid (tiles, C): class c's keys occupy [c * B*N, c * B*N + |V|), its histogram [c][digit][tile]
__global__ void __launch_bounds__(kSortThreads) occ_hist_kernel(const OccParams p, const uint32_t *keys, int shift) {
    const int c = blockIdx.y;
    radix_tile_hist(keys + c * p.nvox, [&] { return class_count(p, c); }, shift,
                    p.hist + static_cast<long long>(c) * kRadix * p.tiles, p.tiles, blockIdx.x);
}

// The scanned histogram runs over every class: class c's positions start at its first entry, and are moved back to
// the start of its own range
__global__ void __launch_bounds__(kSortThreads) occ_scatter_kernel(const OccParams p, const uint32_t *keys_in,
                                                                   const int *vals_in, uint32_t *keys_out,
                                                                   int *vals_out, int shift) {
    const int c = blockIdx.y;
    const long long n = class_count(p, c);
    const long long t0 = static_cast<long long>(blockIdx.x) * kSortTile;
    if (t0 >= n) return;
    const int *hist = p.hist + static_cast<long long>(c) * kRadix * p.tiles;
    const long long to = c * p.nvox - hist[0];
    radix_tile_scatter(keys_in + c * p.nvox, vals_in + c * p.nvox, keys_out + to, vals_out + to, [n] { return n; },
                       shift, hist, p.tiles, blockIdx.x);
}

// ---------------------------------------------------------------------------------------------------------- lovasz
// Each thread of a tile's block owns kSortIters consecutive sorted entries
__device__ __forceinline__ int sorted_fg(const OccParams &p, int c, long long k, long long n) {
    if (k >= n) return 0;
    const int v = p.vals[0][c * p.nvox + k] & ~static_cast<int>(kNegBit);
    return p.vlab[v] == c ? 1 : 0;
}

__global__ void __launch_bounds__(kSortThreads) occ_fg_count_kernel(const OccParams p) {
    const int c = blockIdx.y;
    const long long n = class_count(p, c);
    const long long k0 = static_cast<long long>(blockIdx.x) * kSortTile + threadIdx.x * kSortIters;
    int s = 0;
    if (k0 < n)
        for (int j = 0; j < kSortIters; ++j) s += sorted_fg(p, c, k0 + j, n);
    int total;
    block_exclusive_scan(s, total);
    if (threadIdx.x == 0) p.fgpart[c * p.tiles + blockIdx.x] = total;
}

template <bool GRAD>
__global__ void __launch_bounds__(kSortThreads) occ_lovasz_kernel(const OccParams p) {
    const int c = blockIdx.y;
    const long long n = class_count(p, c);
    const long long k0 = static_cast<long long>(blockIdx.x) * kSortTile + threadIdx.x * kSortIters;
    int fg[kSortIters], s = 0;
#pragma unroll
    for (int j = 0; j < kSortIters; ++j) {
        fg[j] = sorted_fg(p, c, k0 + j, n);
        s += fg[j];
    }
    int total;
    const int ex = block_exclusive_scan(s, total);
    double acc = 0.0;
    if (k0 < n) {
        const double G = p.fg[c];
        int run = p.fgpart[c * p.tiles + blockIdx.x] - p.fgpart[c * p.tiles] + ex;   // sum fg before entry k0
        // J before entry k: 1 - (G - run) / (G + k - run); J_{-1} = 0
        double j_prev = 1.0 - (G - run) / (G + static_cast<double>(k0) - run);
        for (int j = 0; j < kSortIters && k0 + j < n; ++j) {
            const long long k = k0 + j, at = c * p.nvox + k;
            run += fg[j];
            const double jk = 1.0 - (G - run) / (G + static_cast<double>(k + 1) - run);
            const double delta = jk - j_prev;
            j_prev = jk;
            const double e = __uint_as_float(~p.keys[0][at]);
            acc += e * delta;
            if (GRAD) {
                const int val = p.vals[0][at];
                // d|fg - r| / dr = -sign(fg - r), and 0 where the error is 0 (torch.abs)
                const double d = e == 0.0 ? 0.0 : ((val & static_cast<int>(kNegBit)) ? delta : -delta);
                p.dr[c * p.nvox + (val & ~static_cast<int>(kNegBit))] = d;
            }
        }
    }
    const double t = block_sum(acc);
    if (threadIdx.x == 0) p.lpart[c * p.tiles + blockIdx.x] = t;
}

// ---------------------------------------------------------------------------------------------------------- finish
__global__ void __launch_bounds__(kOccThreads) occ_finish_kernel(const OccParams p, int vox_blocks) {
    double num = 0.0, den = 0.0;
    for (int i = threadIdx.x; i < vox_blocks; i += kOccThreads) {
        num += p.cepart[2 * i];
        den += p.cepart[2 * i + 1];
    }
    num = block_sum(num);
    den = block_sum(den);
    double lov = 0.0;
    int present = 0;
    for (int c = 0; c < p.d.C; ++c) {
        double lc = 0.0;
        for (int t = threadIdx.x; t < p.tiles; t += kOccThreads) lc += p.lpart[c * p.tiles + t];
        lc = block_sum(lc);
        if (p.fg[c] > 0 && p.vpos[p.nvox] > 0) {
            lov += lc;
            ++present;
        }
    }
    if (threadIdx.x == 0) {
        const double ce = num / den;   // NaN for an empty S, as PyTorch's mean
        if (present > 0) lov /= present;
        const double wt = p.d.weight;
        p.loss[0] = __double2float_rn(wt * (static_cast<double>(p.d.ce_weight) * ce +
                                            static_cast<double>(p.d.lovasz_weight) * lov));
        p.loss[1] = __double2float_rn(ce);
        p.loss[2] = __double2float_rn(lov);
        p.head->ce_scale = wt * static_cast<double>(p.d.ce_weight) / den;
        p.head->lov_scale = present > 0 ? wt * static_cast<double>(p.d.lovasz_weight) / present : 0.0;
    }
}

// ---------------------------------------------------------------------------------------------------------- grad
template <int C, bool PROBS>
__global__ void __launch_bounds__(kOccThreads) occ_grad_kernel(const OccParams p) {
    const long long i = static_cast<long long>(blockIdx.x) * kOccThreads + threadIdx.x;
    if (i >= p.nvox) return;
    const long long b = i / p.d.N, n = i - b * p.d.N;
    float *g_out = p.grad + b * p.sb + n * p.sn;
    const Voxel v = classify(p, i);
    double g[C];
#pragma unroll
    for (int c = 0; c < C; ++c) g[c] = 0.0;
    if (v.in_s) {
        const float *x = p.pred + b * p.sb + n * p.sn;
        double r[C];
#pragma unroll
        for (int c = 0; c < C; ++c) r[c] = __ldg(x + c * p.sc);
        if (!PROBS) {
            double m = r[0];
#pragma unroll
            for (int c = 1; c < C; ++c) m = fmax(m, r[c]);
            double s = 0.0;
#pragma unroll
            for (int c = 0; c < C; ++c) {
                r[c] = exp(r[c] - m);
                s += r[c];
            }
#pragma unroll
            for (int c = 0; c < C; ++c) r[c] /= s;
        }
        if (v.in_v && p.head->lov_scale != 0.0) {
            const int at = p.vpos[i];
            const double ls = p.head->lov_scale;
            double dr[C], dot = 0.0;
#pragma unroll
            for (int c = 0; c < C; ++c) {
                dr[c] = __ldg(p.fg + c) > 0 ? ls * p.dr[c * p.nvox + at] : 0.0;
                dot += dr[c] * r[c];
            }
#pragma unroll
            for (int c = 0; c < C; ++c) g[c] = PROBS ? dr[c] : r[c] * (dr[c] - dot);
        }
        if (has_class(p, v.y) && v.y != p.d.ignore_index) {
            const int y = static_cast<int>(v.y);
            const double sw = p.head->ce_scale * static_cast<double>(__ldg(p.w + y));
#pragma unroll
            for (int c = 0; c < C; ++c) {
                if (PROBS) {
                    if (c != y) continue;
                    // d(-log clamp(x))/dx = -1 / clamp(x) where lo <= x <= hi (torch.clamp passes the bounds), else 0
                    const float xy = static_cast<float>(r[c]);
                    if (xy >= kProbLo && xy <= kProbHi) g[c] -= sw / static_cast<double>(xy);
                } else {
                    g[c] += sw * (r[c] - (c == y ? 1.0 : 0.0));
                }
            }
        }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) g_out[c * p.sc] = __double2float_rn(g[c]);
}

int check_occ_desc(const gf_occ_loss_desc *d) {
    GF_REQUIRE(d != nullptr, GF_ERR_INVALID_ARG, "occ loss: desc is NULL");
    GF_REQUIRE(d->batch >= 0 && d->N >= 0, GF_ERR_INVALID_ARG, "occ loss: negative batch=%d or N=%d", d->batch, d->N);
    GF_REQUIRE(d->branch == GF_OCC_LOGITS || d->branch == GF_OCC_PROBS, GF_ERR_INVALID_ARG,
               "occ loss: unknown branch %d (GF_OCC_LOGITS = 0, GF_OCC_PROBS = 1)", d->branch);
    GF_REQUIRE(d->layout == GF_OCC_VOXEL_MAJOR || d->layout == GF_OCC_CLASS_MAJOR, GF_ERR_INVALID_ARG,
               "occ loss: unknown layout %d (GF_OCC_VOXEL_MAJOR = 0, GF_OCC_CLASS_MAJOR = 1)", d->layout);
    const int rc = dispatch_classes(d->C, "occ loss", [](auto) { return GF_OK; });
    if (rc != GF_OK) return rc;
    OccPlan pl;
    return occ_plan(*d, pl);
}

OccParams occ_params(const gf_occ_loss_desc &d, const OccPlan &pl, const float *pred, const int64_t *labels,
                     const uint8_t *mask, const float *w, float *loss, float *grad, void *workspace) {
    OccParams p{};
    p.d = d;
    p.nvox = pl.nvox;
    p.tiles = pl.tiles;
    const long long N = d.N, C = d.C;
    p.sb = N * C;
    p.sc = d.layout == GF_OCC_VOXEL_MAJOR ? 1 : N;
    p.sn = d.layout == GF_OCC_VOXEL_MAJOR ? C : 1;
    p.pred = pred; p.labels = labels; p.mask = mask; p.w = w; p.loss = loss; p.grad = grad;
    char *ws = static_cast<char *>(workspace);
    p.head = reinterpret_cast<OccHead *>(ws + pl.head);
    p.fg = reinterpret_cast<int *>(ws + pl.fg);
    p.vpos = reinterpret_cast<int *>(ws + pl.vpos);
    p.vlab = reinterpret_cast<uint8_t *>(ws + pl.vlab);
    for (int i = 0; i < 2; ++i) {
        p.keys[i] = reinterpret_cast<uint32_t *>(ws + pl.pair[i]);
        p.vals[i] = reinterpret_cast<int *>(ws + pl.pair[i] + pl.cv * sizeof(uint32_t));
    }
    p.dr = reinterpret_cast<double *>(ws + pl.pair[1]);
    p.hist = reinterpret_cast<int *>(ws + pl.hist);
    p.fgpart = reinterpret_cast<int *>(ws + pl.fgpart);
    p.lpart = reinterpret_cast<double *>(ws + pl.lpart);
    p.cepart = reinterpret_cast<double *>(ws + pl.cepart);
    return p;
}

template <int C, bool PROBS>
int launch_occ_loss(const OccParams &p, const OccPlan &pl, int *partials, cudaStream_t stream) {
    GF_CUDA_TRY(cudaMemsetAsync(p.head, 0, pl.vpos - pl.head, stream));   // head and the foreground counts
    occ_select_kernel<<<pl.vox_blocks, kOccThreads, 0, stream>>>(p);
    int e = exclusive_scan(p.vpos, pl.nvox + 1, partials, stream);
    if (e != GF_OK) return e;
    occ_keys_kernel<C, PROBS><<<pl.vox_blocks, kOccThreads, 0, stream>>>(p);
    const dim3 grid(pl.tiles, C);
    int cur = 0;
    for (int shift = 0; shift < 32; shift += kRadixBits, cur ^= 1) {
        occ_hist_kernel<<<grid, kSortThreads, 0, stream>>>(p, p.keys[cur], shift);
        e = exclusive_scan(p.hist, static_cast<long long>(kRadix) * pl.tiles * C, partials, stream);
        if (e != GF_OK) return e;
        occ_scatter_kernel<<<grid, kSortThreads, 0, stream>>>(p, p.keys[cur], p.vals[cur], p.keys[cur ^ 1],
                                                              p.vals[cur ^ 1], shift);
    }
    // four passes: the sorted keys and values are back in pair[0], and pair[1] is free for dL/dr
    occ_fg_count_kernel<<<grid, kSortThreads, 0, stream>>>(p);
    e = exclusive_scan(p.fgpart, static_cast<long long>(C) * pl.tiles, partials, stream);
    if (e != GF_OK) return e;
    if (p.grad)
        occ_lovasz_kernel<true><<<grid, kSortThreads, 0, stream>>>(p);
    else
        occ_lovasz_kernel<false><<<grid, kSortThreads, 0, stream>>>(p);
    occ_finish_kernel<<<1, kOccThreads, 0, stream>>>(p, pl.vox_blocks);
    if (p.grad) occ_grad_kernel<C, PROBS><<<pl.vox_blocks, kOccThreads, 0, stream>>>(p);
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}

}  // namespace
}  // namespace gf

using namespace gf;

extern "C" {

size_t gf_occ_loss_workspace_bytes(const gf_occ_loss_desc *desc) {
    if (check_occ_desc(desc) != GF_OK) return 0;
    OccPlan pl;
    occ_plan(*desc, pl);
    return pl.bytes;
}

int gf_occ_loss(const gf_occ_loss_desc *desc, const float *pred, const int64_t *labels, const uint8_t *mask,
                const float *class_weights, float *loss_out, float *grad_out, void *workspace, size_t workspace_bytes,
                gf_stream_t stream_) {
    int rc = check_occ_desc(desc);
    if (rc != GF_OK) return rc;
    OccPlan pl;
    occ_plan(*desc, pl);
    GF_REQUIRE(loss_out != nullptr && class_weights != nullptr, GF_ERR_INVALID_ARG,
               "occ loss: loss_out / class_weights is NULL");
    if (pl.nvox > 0)
        GF_REQUIRE(pred != nullptr && labels != nullptr, GF_ERR_INVALID_ARG, "occ loss: pred / labels is NULL");
    GF_REQUIRE(workspace != nullptr && workspace_bytes >= pl.bytes, GF_ERR_WORKSPACE,
               "occ loss: workspace too small (%zu < %zu bytes)", workspace_bytes, pl.bytes);
    GF_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & (kOccAlign - 1)) == 0, GF_ERR_WORKSPACE,
               "occ loss: workspace must be 256-byte aligned");
    const OccParams p = occ_params(*desc, pl, pred, labels, mask, class_weights, loss_out, grad_out, workspace);
    int *partials = reinterpret_cast<int *>(static_cast<char *>(workspace) + pl.partials);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    return dispatch_classes(desc->C, "occ loss", [&](auto cc) {
        constexpr int C = decltype(cc)::value;
        return desc->branch == GF_OCC_PROBS ? launch_occ_loss<C, true>(p, pl, partials, stream)
                                            : launch_occ_loss<C, false>(p, pl, partials, stream);
    });
}

int gf_debug_occ_loss_order(const gf_occ_loss_desc *desc, const void *workspace, gf_stream_t stream_,
                            int32_t *host_order, int32_t *host_num_v, uint8_t *host_present) {
    int rc = check_occ_desc(desc);
    if (rc != GF_OK) return rc;
    GF_REQUIRE(workspace && host_order && host_num_v && host_present, GF_ERR_INVALID_ARG,
               "occ loss order: NULL argument");
    OccPlan pl;
    occ_plan(*desc, pl);
    const char *ws = static_cast<const char *>(workspace);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int fg[kMaxClasses];
    GF_CUDA_TRY(cudaMemcpyAsync(host_num_v, ws + pl.vpos + pl.nvox * sizeof(int), sizeof(int),
                                cudaMemcpyDeviceToHost, stream));
    GF_CUDA_TRY(cudaMemcpyAsync(fg, ws + pl.fg, desc->C * sizeof(int), cudaMemcpyDeviceToHost, stream));
    GF_CUDA_TRY(cudaStreamSynchronize(stream));
    const int nv = *host_num_v;
    const int *vals = reinterpret_cast<const int *>(ws + pl.pair[0] + pl.cv * sizeof(uint32_t));
    for (int c = 0; c < desc->C; ++c) {
        host_present[c] = fg[c] > 0 && nv > 0 ? 1 : 0;
        if (host_present[c])
            GF_CUDA_TRY(cudaMemcpyAsync(host_order + c * pl.nvox, vals + c * pl.nvox, nv * sizeof(int),
                                        cudaMemcpyDeviceToHost, stream));
    }
    GF_CUDA_TRY(cudaStreamSynchronize(stream));
    for (int c = 0; c < desc->C; ++c)
        if (host_present[c])
            for (int k = 0; k < nv; ++k) host_order[c * pl.nvox + k] &= ~static_cast<int32_t>(kNegBit);
    return GF_OK;
}

}  // extern "C"
