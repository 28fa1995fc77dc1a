// Submanifold sparse convolution (gf_subm_conv_*): spconv's SubMConv3d as the encoder's SparseConv3D calls it
// (model/encoder/gaussian_encoder/spconv3d_module.py:10-83), forward and backward, with C = c_in = c_out = 128.
//
// Rulebook (from the indices alone; every step is integer work, so its result does not depend on the launch):
//   1. rows     per row: validity (status bit otherwise), atomicMin(row) into a dense voxel table [B, X, Y, Z]
//   2. scan     exclusive integer scan of the occupied flags: slot = the voxel's place among the occupied voxels in
//               (b, x, y, z) order, M = their count; the table then maps voxel -> slot, rep[slot] = its lowest row
//   3. nbr      per (offset, slot): the neighbour's slot or -1, as nbr[o][slot] ([K][N], K = k^3); an integer scan of
//               the hits gives the per-offset pair lists (the slots with a neighbour at o, ascending)
//   4. sort     the rows by slot with the stable radix sort of radix_sort.cuh: the rows of a voxel, ascending
//
// Forward, per call: acc[slot] = bias; then for o = 0 .. K-1 in turn, one launch adds
// acc[v] += W_o . features[rep(nbr[o][v])] over o's pairs.  A voxel has at most one neighbour per offset, so the adds
// of one launch never meet, and the launches run in offset order: every output is the same fixed-order fp32 sum on
// every call, without atomics.  Each row then reads its voxel's acc (0 for an invalid row).
//
// Backward: dYsum[slot] = the sum of grad_out over the voxel's rows, ascending.  grad_features runs the forward's
// chain on dYsum with the mirrored weights W_{K-1-o}^T (delta_{K-1-o} = -delta_o), written to representative rows.
// grad_weight: dW_o = sum over o's pairs of dYsum[v]^T x[rep(nbr[o][v])], in GF_SUBM_DW_PIECES fixed pieces of the pair
// list summed in piece order.  grad_bias: fixed block partials of dYsum summed in block order.
#include <algorithm>
#include <vector>

#include "gf_b200_debug.h"
#include "radix_sort.cuh"

namespace gf {
namespace {

constexpr int kSubmC = 128;                 // c_in = c_out: the only width the encoder uses
constexpr int kSubmThreads = 256;
constexpr int kGemmRows = 64;               // pairs per CTA of the per-offset GEMM
constexpr int kDwRows = 32;                 // pairs per staged chunk of the weight-gradient kernel
constexpr int kBiasPieces = 64;
constexpr size_t kSubmAlign = 256;
constexpr int kEmpty = 0x7f7f7f7f;          // voxel-table sentinel (memset byte 0x7f), above every row index
constexpr size_t kGemmSmem = sizeof(float) * (kSubmC * kGemmRows + kSubmC * kSubmC);

struct SubmHead {
    uint32_t status;   // GF_FLAG_INDEX_OUT_OF_RANGE
};

// Workspace of one desc; see the formula in gf_b200.h.  `acc` doubles as the rulebook's scratch for the pair scan.
struct SubmPlan {
    long long nvox, nk;    // B*X*Y*Z, K*N
    int K, tiles, passes;
    size_t head, table, vslot, rep, svox, row_slot, keys[2], vals[2], seg, hist, nbr, pairs, off, partials, acc,
        dysum, wpack, dwpart, bpart, bytes;
};

int subm_plan(const gf_subm_conv_desc &d, SubmPlan &pl) {
    const long long N = d.num_rows;
    pl.nvox = 1;   // step by step, each factor < 2^31, so the product cannot overflow before the check
    for (const int f : {d.batch, d.X, d.Y, d.Z}) {
        pl.nvox *= f;
        GF_REQUIRE(pl.nvox < (1ll << 31), GF_ERR_UNSUPPORTED, "subm conv: B*X*Y*Z >= 2^31 voxels, the op takes < 2^31");
    }
    pl.K = d.kernel_size * d.kernel_size * d.kernel_size;
    pl.nk = N * pl.K;
    GF_REQUIRE(pl.nk < (1ll << 31), GF_ERR_UNSUPPORTED, "subm conv: N*k^3 = %lld, the op takes < 2^31", pl.nk);
    GF_REQUIRE(N * kSubmC < (1ll << 31), GF_ERR_UNSUPPORTED, "subm conv: N*C = %lld, the op takes < 2^31", N * kSubmC);
    pl.tiles = static_cast<int>((N + kSortTile - 1) / kSortTile);
    pl.passes = 0;   // sort keys are slots in [0, N] (N: an invalid row)
    while (pl.passes < 4 && (N >> (kRadixBits * pl.passes)) > 0) ++pl.passes;
    const long long hist = static_cast<long long>(kRadix) * pl.tiles;
    size_t off = 0;
    auto take = [&](long long count, size_t elem) {
        const size_t at = off;
        off += (static_cast<size_t>(count) * elem + kSubmAlign - 1) / kSubmAlign * kSubmAlign;
        return at;
    };
    pl.head = take(1, sizeof(SubmHead));
    pl.table = take(pl.nvox, sizeof(int));
    pl.vslot = take(pl.nvox + 1, sizeof(int));
    pl.rep = take(N, sizeof(int));
    pl.svox = take(N, sizeof(int));
    pl.row_slot = take(N, sizeof(int));
    for (int i = 0; i < 2; ++i) {
        pl.keys[i] = take(N, sizeof(uint32_t));
        pl.vals[i] = take(N, sizeof(int));
    }
    pl.seg = take(N + 1, sizeof(int));
    pl.hist = take(hist, sizeof(int));
    pl.nbr = take(pl.nk, sizeof(int));
    pl.pairs = take(pl.nk, sizeof(int));
    pl.off = take(pl.K + 1, sizeof(int));
    pl.partials = take(scan_partials_count(std::max({pl.nvox + 1, pl.nk + 1, hist})), sizeof(int));
    pl.acc = take(N * kSubmC, sizeof(float));   // >= nk + 1 ints: the pair scan's scratch in the rulebook
    pl.dysum = take(N * kSubmC, sizeof(float));
    pl.wpack = take(static_cast<long long>(pl.K) * kSubmC * kSubmC, sizeof(float));
    pl.dwpart = take(static_cast<long long>(pl.K) * GF_SUBM_DW_PIECES * kSubmC * kSubmC, sizeof(float));
    pl.bpart = take(static_cast<long long>(kBiasPieces) * kSubmC, sizeof(float));
    pl.bytes = off;
    return GF_OK;
}

struct SubmParams {
    int B, X, Y, Z, k, K, N;
    long long nvox;
    SubmHead *head;
    int *table, *vslot, *rep, *svox, *row_slot, *seg, *nbr, *pairs, *off, *hist;
    uint32_t *keys[2];
    int *vals[2];
    int *scratch;             // rulebook: K*N + 1 ints of pair flags / positions (aliases acc)
    float *acc, *dysum, *wpack, *dwpart, *bpart;
};

SubmParams subm_params(const gf_subm_conv_desc &d, const SubmPlan &pl, void *workspace) {
    SubmParams p{};
    p.B = d.batch; p.X = d.X; p.Y = d.Y; p.Z = d.Z; p.k = d.kernel_size; p.K = pl.K; p.N = d.num_rows;
    p.nvox = pl.nvox;
    char *ws = static_cast<char *>(workspace);
    auto at = [ws](size_t o) { return reinterpret_cast<int *>(ws + o); };
    p.head = reinterpret_cast<SubmHead *>(ws + pl.head);
    p.table = at(pl.table); p.vslot = at(pl.vslot); p.rep = at(pl.rep); p.svox = at(pl.svox);
    p.row_slot = at(pl.row_slot); p.seg = at(pl.seg); p.nbr = at(pl.nbr); p.pairs = at(pl.pairs);
    p.off = at(pl.off); p.hist = at(pl.hist);
    for (int i = 0; i < 2; ++i) {
        p.keys[i] = reinterpret_cast<uint32_t *>(ws + pl.keys[i]);
        p.vals[i] = at(pl.vals[i]);
    }
    p.scratch = at(pl.acc);
    p.acc = reinterpret_cast<float *>(ws + pl.acc);
    p.dysum = reinterpret_cast<float *>(ws + pl.dysum);
    p.wpack = reinterpret_cast<float *>(ws + pl.wpack);
    p.dwpart = reinterpret_cast<float *>(ws + pl.dwpart);
    p.bpart = reinterpret_cast<float *>(ws + pl.bpart);
    return p;
}

__device__ __forceinline__ int num_slots(const SubmParams &p) { return p.vslot[p.nvox]; }

inline unsigned blocks_for(long long n, int per) { return static_cast<unsigned>((n + per - 1) / per); }

// ---------------------------------------------------------------------------------------------------------- rulebook
__global__ void __launch_bounds__(kSubmThreads) subm_rows_kernel(const SubmParams p, const int32_t *indices) {
    const int i = blockIdx.x * kSubmThreads + threadIdx.x;
    if (i >= p.N) return;
    const int4 r = reinterpret_cast<const int4 *>(indices)[i];
    if (r.x < 0 || r.x >= p.B || r.y < 0 || r.y >= p.X || r.z < 0 || r.z >= p.Y || r.w < 0 || r.w >= p.Z) {
        atomicOr(&p.head->status, GF_FLAG_INDEX_OUT_OF_RANGE);
        return;
    }
    const long long v = ((static_cast<long long>(r.x) * p.X + r.y) * p.Y + r.z) * p.Z + r.w;
    atomicMin(p.table + v, i);
}

__global__ void __launch_bounds__(kSubmThreads) subm_occupied_kernel(const SubmParams p) {
    const long long v = static_cast<long long>(blockIdx.x) * kSubmThreads + threadIdx.x;
    if (v < p.nvox) p.vslot[v] = p.table[v] != kEmpty ? 1 : 0;
    if (v == 0) p.vslot[p.nvox] = 0;
}

// after the scan: rep and voxel of every slot; the table now maps an occupied voxel to its slot
__global__ void __launch_bounds__(kSubmThreads) subm_slots_kernel(const SubmParams p) {
    const long long v = static_cast<long long>(blockIdx.x) * kSubmThreads + threadIdx.x;
    if (v >= p.nvox) return;
    const int r = p.table[v];
    if (r == kEmpty) return;
    const int s = p.vslot[v];
    p.rep[s] = r;
    p.svox[s] = static_cast<int>(v);
    p.table[v] = s;
}

// slot of every row and the sort's input (key = slot, N for an invalid row)
__global__ void __launch_bounds__(kSubmThreads) subm_row_slot_kernel(const SubmParams p, const int32_t *indices) {
    const int i = blockIdx.x * kSubmThreads + threadIdx.x;
    if (i >= p.N) return;
    const int4 r = reinterpret_cast<const int4 *>(indices)[i];
    int s = -1;
    if (r.x >= 0 && r.x < p.B && r.y >= 0 && r.y < p.X && r.z >= 0 && r.z < p.Y && r.w >= 0 && r.w < p.Z)
        s = p.table[((static_cast<long long>(r.x) * p.X + r.y) * p.Y + r.z) * p.Z + r.w];
    p.row_slot[i] = s;
    p.keys[0][i] = s < 0 ? static_cast<uint32_t>(p.N) : static_cast<uint32_t>(s);
    p.vals[0][i] = i;
}

// grid (N / threads, K): nbr[o][s] and the pair flag at o * N + s
__global__ void __launch_bounds__(kSubmThreads) subm_nbr_kernel(const SubmParams p) {
    const int s = blockIdx.x * kSubmThreads + threadIdx.x;
    const int o = blockIdx.y;
    if (s >= p.N) return;
    int n = -1;
    if (s < num_slots(p)) {
        int v = p.svox[s];
        const int z = v % p.Z; v /= p.Z;
        const int y = v % p.Y; v /= p.Y;
        const int x = v % p.X;
        const int b = v / p.X;
        const int h = (p.k - 1) / 2;
        const int nx = x + o / (p.k * p.k) - h, ny = y + (o / p.k) % p.k - h, nz = z + o % p.k - h;
        if (nx >= 0 && nx < p.X && ny >= 0 && ny < p.Y && nz >= 0 && nz < p.Z) {
            const int t = p.table[((static_cast<long long>(b) * p.X + nx) * p.Y + ny) * p.Z + nz];
            n = t == kEmpty ? -1 : t;
        }
    }
    const long long at = static_cast<long long>(o) * p.N + s;
    p.nbr[at] = n;
    p.scratch[at] = n >= 0 ? 1 : 0;
    if (s == 0 && o == 0) p.scratch[static_cast<long long>(p.K) * p.N] = 0;
}

// after the scan of the flags: o's pairs at pairs[off[o] .. off[o + 1]), slots ascending
__global__ void __launch_bounds__(kSubmThreads) subm_pairs_kernel(const SubmParams p) {
    const int s = blockIdx.x * kSubmThreads + threadIdx.x;
    const int o = blockIdx.y;
    if (s >= p.N) return;
    const long long at = static_cast<long long>(o) * p.N + s;
    if (p.nbr[at] >= 0) p.pairs[p.scratch[at]] = s;
    if (s == 0) {
        p.off[o] = p.scratch[at];
        if (o == p.K - 1) p.off[p.K] = p.scratch[static_cast<long long>(p.K) * p.N];
    }
}

__global__ void __launch_bounds__(kSortThreads) subm_hist_kernel(const SubmParams p, const uint32_t *keys, int shift) {
    radix_tile_hist(keys, [&] { return static_cast<long long>(p.N); }, shift, p.hist, gridDim.x, blockIdx.x);
}

__global__ void __launch_bounds__(kSortThreads) subm_scatter_kernel(const SubmParams p, const uint32_t *keys_in,
                                                                    const int *vals_in, uint32_t *keys_out,
                                                                    int *vals_out, int shift) {
    radix_tile_scatter(keys_in, vals_in, keys_out, vals_out, [&] { return static_cast<long long>(p.N); }, shift,
                       p.hist, gridDim.x, blockIdx.x);
}

// the rows of slot s are sorted[seg[s] .. seg[s + 1]); seg[M] = the valid row count
__global__ void __launch_bounds__(kSubmThreads) subm_seg_kernel(const SubmParams p, const uint32_t *keys) {
    const int j = blockIdx.x * kSubmThreads + threadIdx.x;
    if (j >= p.N) return;
    const uint32_t key = keys[j];
    if (key >= static_cast<uint32_t>(p.N)) return;
    if (j == 0 || keys[j - 1] != key) p.seg[key] = j;
    if (j == p.N - 1 || keys[j + 1] >= static_cast<uint32_t>(p.N)) p.seg[key + 1] = j + 1;
}

// ---------------------------------------------------------------------------------------------------------- GEMM
// wpack[o] as the [k][n] matrix the GEMM multiplies by: forward B_o[ci][co] = W[co][o][ci]; mirrored (grad_features)
// B_o[co][ci] = W[co][K-1-o][ci].  Grid (C/32, C/32, K), 32 x 8 threads: a 32 x 32 tile of W[:, o', :] is read along
// ci and written along co (forward, a transpose through shared memory) or along ci (mirrored), both coalesced.
constexpr int kPackTile = 32, kPackRows = 8;
template <bool MIRROR>
__global__ void __launch_bounds__(kPackTile * kPackRows) subm_pack_weight_kernel(const SubmParams p, const float *w) {
    __shared__ float tile[kPackTile][kPackTile + 1];
    const int o = blockIdx.z, src_o = MIRROR ? p.K - 1 - o : o;
    const int co0 = blockIdx.y * kPackTile, ci0 = blockIdx.x * kPackTile;
    const int tx = threadIdx.x % kPackTile, ty = threadIdx.x / kPackTile;
    for (int r = ty; r < kPackTile; r += kPackRows)
        tile[r][tx] = __ldg(w + (static_cast<long long>(co0 + r) * p.K + src_o) * kSubmC + ci0 + tx);   // [co][ci]
    __syncthreads();
    float *dst = p.wpack + static_cast<long long>(o) * kSubmC * kSubmC;
    for (int r = ty; r < kPackTile; r += kPackRows) {
        if (MIRROR)
            dst[(co0 + r) * kSubmC + ci0 + tx] = tile[r][tx];
        else
            dst[(ci0 + r) * kSubmC + co0 + tx] = tile[tx][r];
    }
}

int launch_pack_weight(const SubmParams &p, const float *w, bool mirror, cudaStream_t stream) {
    const dim3 grid(kSubmC / kPackTile, kSubmC / kPackTile, p.K);
    if (mirror)
        subm_pack_weight_kernel<true><<<grid, kPackTile * kPackRows, 0, stream>>>(p, w);
    else
        subm_pack_weight_kernel<false><<<grid, kPackTile * kPackRows, 0, stream>>>(p, w);
    return GF_OK;
}

// acc[s] = bias (or 0) for every slot
__global__ void __launch_bounds__(kSubmThreads) subm_init_acc_kernel(const SubmParams p, const float *bias) {
    const long long i = static_cast<long long>(blockIdx.x) * kSubmThreads + threadIdx.x;
    if (i >= static_cast<long long>(num_slots(p)) * kSubmC) return;
    p.acc[i] = bias ? bias[i % kSubmC] : 0.f;
}

// Offset o: acc[v] += src[map(nbr[o][v])] . wpack[o] over o's pairs, kGemmRows pairs per CTA.  The CTA stages the
// gathered rows transposed (As[k][row]) and the whole 128 x 128 matrix (Bs[k][n]); thread (ty, tx) owns rows
// 4 ty .. 4 ty + 3 and columns 4 tx .. 4 tx + 3, 64 + 4 tx .. 64 + 4 tx + 3, and sums k in ascending order.
__global__ void __launch_bounds__(kSubmThreads) subm_gemm_kernel(const SubmParams p, int o, const float *src,
                                                                 const int *src_map) {
    extern __shared__ float4 smem4[];
    float *As = reinterpret_cast<float *>(smem4);    // [kSubmC][kGemmRows]
    float *Bs = As + kSubmC * kGemmRows;             // [kSubmC][kSubmC]
    __shared__ int s_dst[kGemmRows], s_src[kGemmRows];
    const int begin = p.off[o], end = p.off[o + 1];
    const int base = begin + blockIdx.x * kGemmRows;
    if (base >= end) return;
    const int n = min(kGemmRows, end - base);
    const int tid = threadIdx.x;
    if (tid < kGemmRows) {
        int d = -1, s = -1;
        if (tid < n) {
            d = p.pairs[base + tid];
            s = p.nbr[static_cast<long long>(o) * p.N + d];
            if (src_map) s = src_map[s];
        }
        s_dst[tid] = d;
        s_src[tid] = s;
    }
    const float4 *b4 = reinterpret_cast<const float4 *>(p.wpack + static_cast<long long>(o) * kSubmC * kSubmC);
    for (int i = tid; i < kSubmC * kSubmC / 4; i += kSubmThreads) reinterpret_cast<float4 *>(Bs)[i] = __ldg(b4 + i);
    __syncthreads();
    for (int i = tid; i < kGemmRows * kSubmC / 4; i += kSubmThreads) {
        const int r = i % kGemmRows, k4 = i / kGemmRows;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < n) v = __ldg(reinterpret_cast<const float4 *>(src + static_cast<long long>(s_src[r]) * kSubmC) + k4);
        As[(4 * k4 + 0) * kGemmRows + r] = v.x;
        As[(4 * k4 + 1) * kGemmRows + r] = v.y;
        As[(4 * k4 + 2) * kGemmRows + r] = v.z;
        As[(4 * k4 + 3) * kGemmRows + r] = v.w;
    }
    __syncthreads();
    const int ty = tid / 16, tx = tid % 16;
    if (4 * ty >= n) return;   // no barrier follows
    float c[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) c[i][j] = 0.f;
#pragma unroll 4
    for (int k = 0; k < kSubmC; ++k) {
        const float4 a = *reinterpret_cast<const float4 *>(As + k * kGemmRows + 4 * ty);
        const float4 b0 = *reinterpret_cast<const float4 *>(Bs + k * kSubmC + 4 * tx);
        const float4 b1 = *reinterpret_cast<const float4 *>(Bs + k * kSubmC + 64 + 4 * tx);
        const float av[4] = {a.x, a.y, a.z, a.w};
        const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) c[i][j] = fmaf(av[i], bv[j], c[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = 4 * ty + i;
        if (r >= n) break;
        float4 *dst = reinterpret_cast<float4 *>(p.acc + static_cast<long long>(s_dst[r]) * kSubmC);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float4 v = dst[16 * h + tx];
            v.x += c[i][4 * h + 0]; v.y += c[i][4 * h + 1]; v.z += c[i][4 * h + 2]; v.w += c[i][4 * h + 3];
            dst[16 * h + tx] = v;
        }
    }
}

// per row: the voxel's acc; REP_ONLY (grad_features): only at the representative row.  0 everywhere else
template <bool REP_ONLY>
__global__ void __launch_bounds__(kSubmThreads) subm_write_rows_kernel(const SubmParams p, float *out) {
    const long long i = static_cast<long long>(blockIdx.x) * kSubmThreads + threadIdx.x;   // float4 of row i / 32
    if (i >= static_cast<long long>(p.N) * (kSubmC / 4)) return;
    const int row = static_cast<int>(i / (kSubmC / 4)), q = static_cast<int>(i % (kSubmC / 4));
    const int s = p.row_slot[row];
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (s >= 0 && (!REP_ONLY || p.rep[s] == row))
        v = reinterpret_cast<const float4 *>(p.acc + static_cast<long long>(s) * kSubmC)[q];
    reinterpret_cast<float4 *>(out)[i] = v;
}

// ---------------------------------------------------------------------------------------------------------- backward
// one warp per slot: dysum[s] = grad_out summed over the slot's rows, ascending
__global__ void __launch_bounds__(kSubmThreads) subm_dysum_kernel(const SubmParams p, const int *sorted_rows,
                                                                  const float *grad_out) {
    const int s = blockIdx.x * (kSubmThreads / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
    if (s >= num_slots(p)) return;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = p.seg[s]; j < p.seg[s + 1]; ++j) {
        const float4 g = __ldg(reinterpret_cast<const float4 *>(grad_out + static_cast<long long>(sorted_rows[j]) * kSubmC) + lane);
        acc.x += g.x; acc.y += g.y; acc.z += g.z; acc.w += g.w;
    }
    reinterpret_cast<float4 *>(p.dysum + static_cast<long long>(s) * kSubmC)[lane] = acc;
}

// grid (GF_SUBM_DW_PIECES, K): piece q of o's pair list, dwpart[o][q][co][ci] = sum_j dysum[v_j][co] x[rep(n_j)][ci];
// thread (ty, tx) owns co in {4 ty + i, 64 + 4 ty + i} by ci in {4 tx + j, 64 + 4 tx + j}, j ascending
__global__ void __launch_bounds__(kSubmThreads) subm_dw_kernel(const SubmParams p, const float *x) {
    __shared__ __align__(16) float Ys[kDwRows][kSubmC], Xs[kDwRows][kSubmC];
    __shared__ int s_dst[kDwRows], s_src[kDwRows];
    const int o = blockIdx.y, q = blockIdx.x, tid = threadIdx.x;
    const int begin = p.off[o], cnt = p.off[o + 1] - begin;
    const int chunk = (cnt + GF_SUBM_DW_PIECES - 1) / GF_SUBM_DW_PIECES;
    const int lo = min(cnt, q * chunk), hi = min(cnt, lo + chunk);
    const int ty = tid / 16, tx = tid % 16;
    float c[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) c[i][j] = 0.f;
    for (int j0 = lo; j0 < hi; j0 += kDwRows) {
        const int n = min(kDwRows, hi - j0);
        if (tid < kDwRows) {
            int d = 0, s = 0;
            if (tid < n) {
                d = p.pairs[begin + j0 + tid];
                s = p.rep[p.nbr[static_cast<long long>(o) * p.N + d]];
            }
            s_dst[tid] = d;
            s_src[tid] = s;
        }
        __syncthreads();
        for (int i = tid; i < kDwRows * kSubmC / 4; i += kSubmThreads) {
            const int r = i / (kSubmC / 4), c4 = i % (kSubmC / 4);
            float4 y = make_float4(0.f, 0.f, 0.f, 0.f), xv = y;
            if (r < n) {
                y = reinterpret_cast<const float4 *>(p.dysum + static_cast<long long>(s_dst[r]) * kSubmC)[c4];
                xv = __ldg(reinterpret_cast<const float4 *>(x + static_cast<long long>(s_src[r]) * kSubmC) + c4);
            }
            reinterpret_cast<float4 *>(&Ys[r][0])[c4] = y;
            reinterpret_cast<float4 *>(&Xs[r][0])[c4] = xv;
        }
        __syncthreads();
        for (int r = 0; r < n; ++r) {
            const float4 a0 = *reinterpret_cast<const float4 *>(&Ys[r][4 * ty]);
            const float4 a1 = *reinterpret_cast<const float4 *>(&Ys[r][64 + 4 * ty]);
            const float4 b0 = *reinterpret_cast<const float4 *>(&Xs[r][4 * tx]);
            const float4 b1 = *reinterpret_cast<const float4 *>(&Xs[r][64 + 4 * tx]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) c[i][j] = fmaf(av[i], bv[j], c[i][j]);
        }
        __syncthreads();
    }
    float *out = p.dwpart + (static_cast<long long>(o) * GF_SUBM_DW_PIECES + q) * kSubmC * kSubmC;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int co = (i < 4 ? 0 : 64) + 4 * ty + (i & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h)
            reinterpret_cast<float4 *>(out + co * kSubmC + 64 * h)[tx] =
                make_float4(c[i][4 * h], c[i][4 * h + 1], c[i][4 * h + 2], c[i][4 * h + 3]);
    }
}

// grad_weight[co][o][ci] = sum over the pieces in order
__global__ void __launch_bounds__(kSubmThreads) subm_dw_reduce_kernel(const SubmParams p, float *grad_weight) {
    const long long i = static_cast<long long>(blockIdx.x) * kSubmThreads + threadIdx.x;
    if (i >= static_cast<long long>(p.K) * kSubmC * kSubmC) return;
    const int ci = static_cast<int>(i % kSubmC);
    const int o = static_cast<int>((i / kSubmC) % p.K);
    const int co = static_cast<int>(i / (static_cast<long long>(kSubmC) * p.K));
    float s = 0.f;
    for (int q = 0; q < GF_SUBM_DW_PIECES; ++q)
        s += p.dwpart[((static_cast<long long>(o) * GF_SUBM_DW_PIECES + q) * kSubmC + co) * kSubmC + ci];
    grad_weight[i] = s;
}

// block q of kBiasPieces sums dysum over its fixed range of slots; thread = channel
__global__ void __launch_bounds__(kSubmC) subm_bias_partial_kernel(const SubmParams p) {
    const int m = num_slots(p);
    const int chunk = (m + kBiasPieces - 1) / kBiasPieces;
    const int lo = min(m, static_cast<int>(blockIdx.x) * chunk), hi = min(m, lo + chunk);
    float s = 0.f;
    for (int v = lo; v < hi; ++v) s += p.dysum[static_cast<long long>(v) * kSubmC + threadIdx.x];
    p.bpart[blockIdx.x * kSubmC + threadIdx.x] = s;
}

__global__ void __launch_bounds__(kSubmC) subm_bias_finish_kernel(const SubmParams p, float *grad_bias) {
    float s = 0.f;
    for (int q = 0; q < kBiasPieces; ++q) s += p.bpart[q * kSubmC + threadIdx.x];
    grad_bias[threadIdx.x] = s;
}

// ---------------------------------------------------------------------------------------------------------- host
int check_subm_desc(const gf_subm_conv_desc *d, SubmPlan &pl) {
    GF_REQUIRE(d != nullptr, GF_ERR_INVALID_ARG, "subm conv: desc is NULL");
    GF_REQUIRE(d->batch >= 1 && d->num_rows >= 1 && d->X >= 1 && d->Y >= 1 && d->Z >= 1, GF_ERR_INVALID_ARG,
               "subm conv: batch=%d, num_rows=%d, X=%d, Y=%d, Z=%d must all be >= 1", d->batch, d->num_rows, d->X,
               d->Y, d->Z);
    GF_REQUIRE(d->kernel_size >= 1 && d->kernel_size <= 5 && d->kernel_size % 2 == 1, GF_ERR_INVALID_ARG,
               "subm conv: kernel_size=%d, the op takes 1, 3 or 5", d->kernel_size);
    GF_REQUIRE(d->c_in == kSubmC && d->c_out == kSubmC, GF_ERR_UNSUPPORTED,
               "subm conv: c_in=%d, c_out=%d; the op is compiled for 128 -> 128", d->c_in, d->c_out);
    return subm_plan(*d, pl);
}

bool aligned16(const void *ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0; }

int check_subm_ws(const SubmPlan &pl, const void *workspace, size_t bytes) {
    GF_REQUIRE(workspace != nullptr && bytes >= pl.bytes, GF_ERR_WORKSPACE,
               "subm conv: workspace too small (%zu < %zu bytes)", bytes, pl.bytes);
    GF_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & (kSubmAlign - 1)) == 0, GF_ERR_WORKSPACE,
               "subm conv: workspace must be 256-byte aligned");
    return GF_OK;
}

// the per-offset chain: acc[v] += src[map(nbr)] . wpack[o], offsets ascending
int launch_offsets(const SubmParams &p, const float *src, const int *src_map, cudaStream_t stream) {
    GF_CUDA_TRY(cudaFuncSetAttribute(subm_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(kGemmSmem)));
    const unsigned grid = blocks_for(p.N, kGemmRows);
    for (int o = 0; o < p.K; ++o) subm_gemm_kernel<<<grid, kSubmThreads, kGemmSmem, stream>>>(p, o, src, src_map);
    return GF_OK;
}

}  // namespace
}  // namespace gf

using namespace gf;

extern "C" {

size_t gf_subm_conv_workspace_bytes(const gf_subm_conv_desc *desc) {
    SubmPlan pl;
    if (check_subm_desc(desc, pl) != GF_OK) return 0;
    return pl.bytes;
}

int gf_subm_conv_rulebook(const gf_subm_conv_desc *desc, const int32_t *indices, void *workspace,
                          size_t workspace_bytes, gf_stream_t stream_) {
    SubmPlan pl;
    int rc = check_subm_desc(desc, pl);
    if (rc != GF_OK) return rc;
    GF_REQUIRE(indices != nullptr, GF_ERR_INVALID_ARG, "subm conv rulebook: indices is NULL");
    GF_REQUIRE(aligned16(indices), GF_ERR_INVALID_ARG,
               "subm conv rulebook: indices must be 16-byte aligned");
    rc = check_subm_ws(pl, workspace, workspace_bytes);
    if (rc != GF_OK) return rc;
    const SubmParams p = subm_params(*desc, pl, workspace);
    int *partials = reinterpret_cast<int *>(static_cast<char *>(workspace) + pl.partials);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const unsigned row_blocks = blocks_for(p.N, kSubmThreads), vox_blocks = blocks_for(pl.nvox, kSubmThreads);
    GF_CUDA_TRY(cudaMemsetAsync(p.head, 0, sizeof(SubmHead), stream));
    GF_CUDA_TRY(cudaMemsetAsync(p.table, 0x7f, pl.nvox * sizeof(int), stream));
    subm_rows_kernel<<<row_blocks, kSubmThreads, 0, stream>>>(p, indices);
    subm_occupied_kernel<<<vox_blocks, kSubmThreads, 0, stream>>>(p);
    rc = exclusive_scan(p.vslot, pl.nvox + 1, partials, stream);
    if (rc != GF_OK) return rc;
    subm_slots_kernel<<<vox_blocks, kSubmThreads, 0, stream>>>(p);
    subm_row_slot_kernel<<<row_blocks, kSubmThreads, 0, stream>>>(p, indices);
    const dim3 nbr_grid(row_blocks, pl.K);
    subm_nbr_kernel<<<nbr_grid, kSubmThreads, 0, stream>>>(p);
    rc = exclusive_scan(p.scratch, pl.nk + 1, partials, stream);
    if (rc != GF_OK) return rc;
    subm_pairs_kernel<<<nbr_grid, kSubmThreads, 0, stream>>>(p);
    int cur = 0;
    for (int pass = 0; pass < pl.passes; ++pass, cur ^= 1) {
        subm_hist_kernel<<<pl.tiles, kSortThreads, 0, stream>>>(p, p.keys[cur], pass * kRadixBits);
        rc = exclusive_scan(p.hist, static_cast<long long>(kRadix) * pl.tiles, partials, stream);
        if (rc != GF_OK) return rc;
        subm_scatter_kernel<<<pl.tiles, kSortThreads, 0, stream>>>(p, p.keys[cur], p.vals[cur], p.keys[cur ^ 1],
                                                                   p.vals[cur ^ 1], pass * kRadixBits);
    }
    // the sorted rows end in pair `cur`; the backward finds them through seg and sorted_rows()
    subm_seg_kernel<<<row_blocks, kSubmThreads, 0, stream>>>(p, p.keys[cur]);
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}

int gf_subm_conv_forward(const gf_subm_conv_desc *desc, void *workspace, const float *features, const float *weight,
                         const float *bias, float *out, gf_stream_t stream_) {
    SubmPlan pl;
    int rc = check_subm_desc(desc, pl);
    if (rc != GF_OK) return rc;
    GF_REQUIRE(features && weight && out, GF_ERR_INVALID_ARG, "subm conv forward: features / weight / out is NULL");
    GF_REQUIRE(aligned16(features) && aligned16(out), GF_ERR_INVALID_ARG,
               "subm conv forward: features and out must be 16-byte aligned (the kernels use 16-byte vector accesses)");
    rc = check_subm_ws(pl, workspace, pl.bytes);
    if (rc != GF_OK) return rc;
    const SubmParams p = subm_params(*desc, pl, workspace);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    launch_pack_weight(p, weight, false, stream);
    subm_init_acc_kernel<<<blocks_for(static_cast<long long>(p.N) * kSubmC, kSubmThreads), kSubmThreads, 0, stream>>>(
        p, bias);
    rc = launch_offsets(p, features, p.rep, stream);
    if (rc != GF_OK) return rc;
    subm_write_rows_kernel<false><<<blocks_for(static_cast<long long>(p.N) * kSubmC / 4, kSubmThreads), kSubmThreads,
                                    0, stream>>>(p, out);
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}

int gf_subm_conv_backward(const gf_subm_conv_desc *desc, void *workspace, const float *features, const float *weight,
                          const float *grad_out, float *grad_features, float *grad_weight, float *grad_bias,
                          gf_stream_t stream_) {
    SubmPlan pl;
    int rc = check_subm_desc(desc, pl);
    if (rc != GF_OK) return rc;
    GF_REQUIRE(grad_out != nullptr, GF_ERR_INVALID_ARG, "subm conv backward: grad_out is NULL");
    GF_REQUIRE(!grad_features || weight, GF_ERR_INVALID_ARG, "subm conv backward: grad_features needs weight");
    GF_REQUIRE(!grad_weight || features, GF_ERR_INVALID_ARG, "subm conv backward: grad_weight needs features");
    GF_REQUIRE(aligned16(features) && aligned16(grad_out) && aligned16(grad_features), GF_ERR_INVALID_ARG,
               "subm conv backward: features, grad_out and grad_features must be 16-byte aligned (the kernels use "
               "16-byte vector accesses)");
    rc = check_subm_ws(pl, workspace, pl.bytes);
    if (rc != GF_OK) return rc;
    const SubmParams p = subm_params(*desc, pl, workspace);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const int *sorted_rows = p.vals[pl.passes & 1];
    subm_dysum_kernel<<<blocks_for(p.N, kSubmThreads / 32), kSubmThreads, 0, stream>>>(p, sorted_rows, grad_out);
    if (grad_features) {
        launch_pack_weight(p, weight, true, stream);
        subm_init_acc_kernel<<<blocks_for(static_cast<long long>(p.N) * kSubmC, kSubmThreads), kSubmThreads, 0,
                               stream>>>(p, nullptr);
        rc = launch_offsets(p, p.dysum, nullptr, stream);
        if (rc != GF_OK) return rc;
        subm_write_rows_kernel<true><<<blocks_for(static_cast<long long>(p.N) * kSubmC / 4, kSubmThreads),
                                       kSubmThreads, 0, stream>>>(p, grad_features);
    }
    if (grad_weight) {
        subm_dw_kernel<<<dim3(GF_SUBM_DW_PIECES, p.K), kSubmThreads, 0, stream>>>(p, features);
        subm_dw_reduce_kernel<<<blocks_for(static_cast<long long>(p.K) * kSubmC * kSubmC, kSubmThreads),
                                kSubmThreads, 0, stream>>>(p, grad_weight);
    }
    if (grad_bias) {
        subm_bias_partial_kernel<<<kBiasPieces, kSubmC, 0, stream>>>(p);
        subm_bias_finish_kernel<<<1, kSubmC, 0, stream>>>(p, grad_bias);
    }
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}

int gf_debug_subm_conv_neighbors(const gf_subm_conv_desc *desc, const void *workspace, gf_stream_t stream_,
                                 int32_t *host_num_voxels, int32_t *host_slot, int32_t *host_rep, int32_t *host_nbr) {
    SubmPlan pl;
    int rc = check_subm_desc(desc, pl);
    if (rc != GF_OK) return rc;
    GF_REQUIRE(workspace && host_num_voxels && host_slot && host_rep && host_nbr, GF_ERR_INVALID_ARG,
               "subm conv neighbours: NULL argument");
    const char *ws = static_cast<const char *>(workspace);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const long long N = desc->num_rows;
    GF_CUDA_TRY(cudaMemcpyAsync(host_num_voxels, ws + pl.vslot + pl.nvox * sizeof(int), sizeof(int),
                                cudaMemcpyDeviceToHost, stream));
    GF_CUDA_TRY(cudaMemcpyAsync(host_slot, ws + pl.row_slot, N * sizeof(int), cudaMemcpyDeviceToHost, stream));
    GF_CUDA_TRY(cudaStreamSynchronize(stream));
    const int m = *host_num_voxels;
    GF_CUDA_TRY(cudaMemcpyAsync(host_rep, ws + pl.rep, m * sizeof(int), cudaMemcpyDeviceToHost, stream));
    // nbr is [K][N] on the device; the host gets [M, K]
    std::vector<int32_t> by_offset(static_cast<size_t>(pl.K) * m);
    if (m > 0)
        GF_CUDA_TRY(cudaMemcpy2DAsync(by_offset.data(), m * sizeof(int), ws + pl.nbr, N * sizeof(int),
                                      m * sizeof(int), pl.K, cudaMemcpyDeviceToHost, stream));
    GF_CUDA_TRY(cudaStreamSynchronize(stream));
    for (int o = 0; o < pl.K; ++o)
        for (int s = 0; s < m; ++s) host_nbr[static_cast<size_t>(s) * pl.K + o] = by_offset[static_cast<size_t>(o) * m + s];
    return GF_OK;
}

}  // extern "C"
