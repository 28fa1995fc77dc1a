// Integer exclusive scan and stable LSD radix sort without CUB, shared by the deterministic deformable-aggregation
// backward (daf_det.cu) and the occupancy loss (occ_loss.cu).  Both results depend on the inputs alone, never on the
// launch: the scan is an integer sum, and the sort places every entry after the equal digits of the entries before it.
//
// One sort pass over a key range is three launches the caller owns:
//   1. radix_tile_hist     per tile of kSortTile keys: the count of every digit, written to hist[digit * tiles + tile]
//   2. exclusive_scan      over the histogram: every (digit, tile) gets its first output position
//   3. radix_tile_scatter  per tile: every entry goes to its digit's position plus the equal digits before it
// The histogram is digit-major within a range, so several ranges laid out one after another ([range][digit][tile])
// are sorted by one scan each pass; a range's positions then start at its first scanned entry.
#pragma once
#include "common.cuh"

namespace gf {
namespace {

constexpr int kScanThreads = 256, kScanItems = 16, kScanTile = kScanThreads * kScanItems;
constexpr int kSortThreads = 256, kSortWarps = kSortThreads / 32, kSortIters = 16;
constexpr int kSortTile = kSortWarps * 32 * kSortIters;   // entries per sort tile; a warp owns 32 * kSortIters of them
constexpr int kRadixBits = 8, kRadix = 1 << kRadixBits;

// ---------------------------------------------------------------------------------------------------------- scans
// Exclusive scan of kScanThreads values of one block; `total` receives their sum.
__device__ __forceinline__ int block_exclusive_scan(int v, int &total) {
    __shared__ int s_warp[kScanThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    int off = 0;
    total = 0;
#pragma unroll
    for (int w = 0; w < kScanThreads / 32; ++w) {
        const int c = s_warp[w];
        if (w < warp) off += c;
        total += c;
    }
    __syncthreads();
    return off + inc - v;
}

__global__ void __launch_bounds__(kScanThreads) scan_reduce_kernel(const int *data, long long n, int *partials) {
    const long long base = static_cast<long long>(blockIdx.x) * kScanTile;
    int s = 0;
    for (int i = threadIdx.x; i < kScanTile; i += kScanThreads)
        if (base + i < n) s += data[base + i];
    int total;
    block_exclusive_scan(s, total);
    if (threadIdx.x == 0) partials[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) scan_partials_kernel(int *partials, int n) {
    int carry = 0;
    for (int base = 0; base < n; base += kScanThreads) {
        const int i = base + threadIdx.x;
        const int v = i < n ? partials[i] : 0;
        int total;
        const int ex = block_exclusive_scan(v, total);
        if (i < n) partials[i] = carry + ex;
        carry += total;
    }
}

__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(int *data, long long n, const int *partials) {
    const long long base = static_cast<long long>(blockIdx.x) * kScanTile + threadIdx.x * kScanItems;
    int v[kScanItems], s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        v[k] = base + k < n ? data[base + k] : 0;
        s += v[k];
    }
    int total;
    int run = partials[blockIdx.x] + block_exclusive_scan(s, total);
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        if (base + k < n) data[base + k] = run;
        run += v[k];
    }
}

// scratch ints exclusive_scan needs for n values
inline long long scan_partials_count(long long n) { return (n + kScanTile - 1) / kScanTile; }

// in place, over n ints (an integer scan: its result does not depend on the launch)
inline int exclusive_scan(int *data, long long n, int *partials, cudaStream_t stream) {
    const long long blocks = (n + kScanTile - 1) / kScanTile;
    scan_reduce_kernel<<<static_cast<unsigned>(blocks), kScanThreads, 0, stream>>>(data, n, partials);
    scan_partials_kernel<<<1, kScanThreads, 0, stream>>>(partials, static_cast<int>(blocks));
    scan_apply_kernel<<<static_cast<unsigned>(blocks), kScanThreads, 0, stream>>>(data, n, partials);
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}

// ---------------------------------------------------------------------------------------------------------- sort
// The key count n of a range is read on the device: count() returns it, and the sort kernels call it where they first
// need it.

// Digit counts of tile `tile` (keys [tile * kSortTile, +kSortTile)) of a range of n keys: hist[digit * tiles + tile].
// A tile at or past n writes zeros.  Every thread of the kSortThreads-thread block calls it.
template <class Count>
__device__ __forceinline__ void radix_tile_hist(const uint32_t *keys, Count count, int shift, int *hist, int tiles,
                                                unsigned tile) {
    __shared__ int cnt[kRadix];
    for (int i = threadIdx.x; i < kRadix; i += kSortThreads) cnt[i] = 0;
    __syncthreads();
    const long long n = count();
    const long long t0 = static_cast<long long>(tile) * kSortTile;
    for (int i = threadIdx.x; i < kSortTile; i += kSortThreads)
        if (t0 + i < n) atomicAdd(&cnt[(keys[t0 + i] >> shift) & (kRadix - 1)], 1);
    __syncthreads();
    for (int dg = threadIdx.x; dg < kRadix; dg += kSortThreads) hist[static_cast<long long>(dg) * tiles + tile] = cnt[dg];
}

// Stable scatter of tile `tile` of a range of n keys (hist as radix_tile_hist wrote it, scanned):
// warp w owns the tile's w-th run of 32 * kSortIters entries.  Pass 1 counts each warp's digits, then every digit's
// start is the tile's scanned offset plus the counts of the warps before; pass 2 places each entry after the equal
// digits of its warp's earlier entries and of the lanes below it (__match_any_sync).  Entry j goes to
// keys_out[position] / vals_out[position].  Every thread of the kSortThreads-thread block calls it.
template <class Count>
__device__ __forceinline__ void radix_tile_scatter(const uint32_t *keys_in, const int *vals_in, uint32_t *keys_out,
                                                   int *vals_out, Count count, int shift, const int *hist,
                                                   int tiles, unsigned tile) {
    __shared__ int wcnt[kSortWarps][kRadix];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long n = count();
    const long long t0 = static_cast<long long>(tile) * kSortTile;
    if (t0 >= n) return;   // uniform over the block
    const long long w0 = t0 + static_cast<long long>(warp) * 32 * kSortIters;
    for (int i = lane; i < kRadix; i += 32) wcnt[warp][i] = 0;
    __syncwarp();
    for (int it = 0; it < kSortIters; ++it) {
        const long long j = w0 + it * 32 + lane;
        const int dg = j < n ? static_cast<int>((keys_in[j] >> shift) & (kRadix - 1)) : kRadix;
        const uint32_t peers = __match_any_sync(0xffffffffu, dg);
        if (dg < kRadix && lane == __ffs(peers) - 1) wcnt[warp][dg] += __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    for (int dg = threadIdx.x; dg < kRadix; dg += kSortThreads) {
        int run = hist[static_cast<long long>(dg) * tiles + tile];
        for (int w = 0; w < kSortWarps; ++w) {
            const int c = wcnt[w][dg];
            wcnt[w][dg] = run;
            run += c;
        }
    }
    __syncthreads();
    for (int it = 0; it < kSortIters; ++it) {
        const long long j = w0 + it * 32 + lane;
        uint32_t key = 0;
        int dg = kRadix;
        if (j < n) {
            key = keys_in[j];
            dg = static_cast<int>((key >> shift) & (kRadix - 1));
        }
        const uint32_t peers = __match_any_sync(0xffffffffu, dg);
        if (dg < kRadix) {
            const int at = wcnt[warp][dg] + __popc(peers & lanemask_lt());
            keys_out[at] = key;
            vals_out[at] = vals_in[j];
        }
        __syncwarp();
        if (dg < kRadix && lane == __ffs(peers) - 1) wcnt[warp][dg] += __popc(peers);
        __syncwarp();
    }
}

}  // namespace
}  // namespace gf
