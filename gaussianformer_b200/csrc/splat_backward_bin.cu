// Splat backward, bin-centric form (replaces BACKWARD::renderCUDA, model/head/localagg/src/backward.cu:24-103 and
// model/head/localagg_prob/src/backward.cu:24-123, for points in canonical voxel order — every shipped config).
//
// The Gaussian-centric kernels (splat_backward.cu) gather one 4C-byte row of the upstream gradient per (Gaussian,
// voxel) pair from L1/L2; ncu shows them waiting on that gather (long scoreboard 3.9 of 8.3 stall cycles per issue, L1
// data pipe 54 %, DRAM 3 %).  Here a CTA owns a bin of 8 x 4 columns x 16 z (the render kernel's bin) and
//
//   * stages the bin's tile of the upstream gradient ([8][4][16][C] fp32 = 36.9 KB for C = 18), its points (6 KB) and,
//     for the prob variant, the per-point terms of prob_aux_kernel (8 KB) into shared memory with TMA tensor copies
//     (cp.async.bulk.tensor.3d, boxes {8C, 4, 8} / {48, 4, 8} / {64, 4, 8} over [B*H][W][D*C]-shaped tensor maps;
//     out-of-grid parts of a box are zero-filled by the hardware) -- every byte of the 46 MB gradient is read from
//     global memory once, coalesced;
//   * resolves the bin's ordered Gaussian list from the supertile list while the copies are in flight (Phase A,
//     resolve_bin_list in common.cuh, shared with the render kernel);
//   * gives every listed Gaussian to EIGHT lanes (four Gaussians per warp at a time; warps take groups of four list
//     entries from a shared counter): the lanes stride over the box clipped to the bin (92 voxels on average for the
//     nuScenes workload -- a whole warp per Gaussian would spend more on its reduction than on the pairs), read their
//     pair's point, gradient row and aux terms from shared memory, accumulate the 28 (+1) sums of GaussAcc, reduce them
//     with a transposing reduction over the eight lanes (28 shuffles for four Gaussians) and add the raw sums to a
//     value-major [32, G] accumulator with one atomic per value;
//   * bin_finish_kernel applies the per-Gaussian linear maps (finish(), splat_bwd_common.cuh) once per Gaussian.
//
// The accumulator is zero-filled by the host first.  Summation order across bins is not fixed (fp32 atomics), so two
// runs may differ in the last bits.  The deterministic route (GF_BWD_DETERMINISTIC: slot_plan_kernel ->
// backward_bin_slots_kernel -> bin_slot_finish_kernel) stores each (Gaussian, bin) sum to its own slot row and adds the
// rows in a fixed order instead.  The Gaussian-centric kernels serve every case this kernel does not cover (points
// not in canonical order, odd strides, misaligned tensors).
#include <cuda.h>

#include "splat_bwd_common.cuh"
#include "splat_host.cuh"

namespace gf {

constexpr int kBinThreads = 256;
constexpr int kBinSeg = 512;      // list entries resolved per segment
// Phase B balance: four list entries share a warp (8 lanes each) and run in lock step, so they should need the same
// number of passes; entries are therefore ordered by key = ceil(volume / 8) with a counting sort, and boxes of
// kWideVol voxels or more (the whole-grid "empty" Gaussian; most Gaussians of the prob config) get a whole warp.
// Host-side model on the nuScenes workload: 667 k -> 372 k warp passes (ideal 339 k).
constexpr int kVolKeys = 64;      // keys 1..64 (a clipped box has at most 512 voxels)
constexpr int kWideVol = 192;

struct alignas(64) BinMaps {
    CUtensorMap grad;   // logits_grad as [B*H][W][D*C]
    CUtensorMap pts;    // pts as [B*H or H][W][D*3]
    CUtensorMap aux;    // prob: aux as [B*H][W][D*4]
};

// Bins (kBinX x kBinY x kBinZ voxels) a Gaussian's clipped box overlaps: a rectangle of nb[0] x nb[1] x nb[2] bins from
// bin b0.  None for an empty box.
struct BoxBins {
    int b0[3], nb[3];
    __device__ __forceinline__ explicit BoxBins(const PackedBox &b) {
        const uint32_t w[3] = {b.x, b.y, b.z};
        const int e[3] = {kBinX, kBinY, kBinZ};
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            b0[a] = static_cast<int>(w[a] & 0xffffu) / e[a];
            nb[a] = b.empty ? 0 : static_cast<int>(w[a] >> 16) / e[a] - b0[a] + 1;
        }
    }
    __device__ __forceinline__ int count() const { return nb[0] * nb[1] * nb[2]; }
};

template <int C, bool PROB>
struct BinSmem {
    // two TMA boxes {8C, 4, 8}: z half h at h*256*C, voxel (x, y, z & 7) at ((x*4 + y)*8 + (z & 7))*C
    alignas(128) float grad[512 * C];
    alignas(128) float pts[512 * 3];                 // one box {48, 4, 8}: (x*4 + y)*48 + z*3
    alignas(128) float4 aux[PROB ? 512 : 1];         // one box {64, 4, 8}: (x*4 + y)*16 + z
    alignas(8) uint2 list[kBinSeg];                  // x: box relative to the bin as bit masks, y: Gaussian index
    alignas(8) uint2 sorted[kBinSeg];                // the same entries ordered by clipped-box volume (counting sort)
    alignas(8) uint64_t bar;
    int warp_count[2][kBinThreads / 32];
    int hist[kVolKeys + 1];                          // counting sort: entries per key, then running offsets
    int n_narrow;                                    // entries served by 8-lane groups (the rest: one warp each)
    int next;                                        // next unclaimed ticket of the segment
};

// Sum of x[i] over the eight lanes of a group for all i at once: afterwards the lane with low bits (b2 b1 b0) holds the
// group totals of x[16*b2 + 8*b1 + 4*b0 + i] in x[i], i = 0..3.  28 shuffles.
__device__ __forceinline__ void group8_transpose_reduce(float x[32], int lane) {
#pragma unroll
    for (int st = 0; st < 3; ++st) {
        const int h = 4 >> st, half = 16 >> st;
        const bool upper = (lane & h) != 0;
#pragma unroll
        for (int i = 0; i < half; ++i) {
            const float send = upper ? x[i] : x[i + half];
            const float keep = upper ? x[i + half] : x[i];
            x[i] = keep + __shfl_xor_sync(0xffffffffu, send, h);
        }
    }
}

__device__ __forceinline__ void tma_load_3d(void *smem_dst, const CUtensorMap *map, int c0, int c1, int c2, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
            smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
        : "memory");
}

// floor(i / n) for 0 <= i < 2048 and 1 <= n <= 16 without a division: i * ceil(2^16 / n) >> 16 (exact: i * (ceil - 2^16/n) < 2^16 / n)
__constant__ uint32_t kRcp16[17] = {0u, 65536u, 32768u, 21846u, 16384u, 13108u, 10923u, 9363u, 8192u,
                                    7282u, 6554u, 5958u, 5462u, 5042u, 4682u, 4370u, 4096u};
__device__ __forceinline__ int small_div(int i, int n) {
    return static_cast<int>((static_cast<uint32_t>(i) * kRcp16[n]) >> 16);
}

// Waits for the bin's tiles, then checks the canonical order of its points (point n must lie in voxel n): the bin
// kernel assumed it; a violation clears the flag, bin_finish_kernel then discards the sums and the Gaussian-centric
// kernels (which build the voxel -> point map) produce the gradients instead.
template <int C, bool PROB>
__device__ __forceinline__ void check_bin_order(const BwdParams &p, BinSmem<C, PROB> &sm, int binX0, int binY0, int binZ0) {
    constexpr int NT = kBinThreads;
    const int tid = threadIdx.x, H = p.d.H, W = p.d.W, D = p.d.D;
    mbar_wait(&sm.bar, 0);
#pragma unroll
    for (int r = 0; r < 512 / NT; ++r) {
        const int i = tid + r * NT, col = i >> 4, z = i & 15;
        const int X = binX0 + (col >> 2), Y = binY0 + (col & 3), Z = binZ0 + z;
        if (X < H && Y < W && Z < D) {
            int vx, vy, vz;
            if (p.in.points_int) {
                const long long n = (static_cast<long long>(X) * W + Y) * D + Z;
                vx = p.in.points_int[3 * n]; vy = p.in.points_int[3 * n + 1]; vz = p.in.points_int[3 * n + 2];
            } else {
                const float *pp = &sm.pts[col * (kBinZ * 3) + z * 3];
                vx = voxel_coord(pp[0], p.d.pc_min[0], p.d.grid_size);
                vy = voxel_coord(pp[1], p.d.pc_min[1], p.d.grid_size);
                vz = voxel_coord(pp[2], p.d.pc_min[2], p.d.grid_size);
            }
            if (vx != X || vy != Y || vz != Z) *p.canon = 0;   // benign race: every writer stores 0
        }
    }
}

// DET (deterministic mode): instead of adding the eight lanes' raw sums to the [32, G] accumulator with atomics, the
// group stores them to the (Gaussian, bin) pair's own slot row, one 16-byte store per lane.  A pair's sums do not
// depend on scheduling: the entry's lanes, strides and wide/narrow choice follow from the entry alone, and the shuffle
// trees are fixed.  With a slot overflow (the route word says so, and the canon flag is already clear) nothing is stored.
// nbx: bins along x (blockIdx.z = sample * nbx + bin x).
template <int C, bool PROB, bool DET>
__device__ __forceinline__ void backward_bin(const BwdParams &pb, int nbx, const BinMaps &maps) {
    constexpr int NT = kBinThreads, CP2 = (C + 1) / 2;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    BinSmem<C, PROB> &sm = *reinterpret_cast<BinSmem<C, PROB> *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int sample = blockIdx.z / nbx;
    const BwdParams p = sample_bwd(pb, sample);
    const int H = p.d.H;
    const int binX0 = (blockIdx.z - sample * nbx) * kBinX, binY0 = blockIdx.y * kBinY, binZ0 = blockIdx.x * kBinZ;
    if (tid == 0) {
        mbar_init(&sm.bar, 1);
        mbar_fence_init();
    }
    pdl_launch_dependents();
    __syncthreads();
    pdl_wait();   // boxes / lists of the preparation kernels, and (transitively) the aux terms of the prob variant

    if (tid == 0) {
        constexpr uint32_t kBytes = 512u * C * 4u + 512u * 3u * 4u + (PROB ? 512u * 16u : 0u);
        mbar_expect_tx(&sm.bar, kBytes);
        const int xr = sample * H + binX0;
        tma_load_3d(&sm.grad[0], &maps.grad, binZ0 * C, binY0, xr, &sm.bar);
        tma_load_3d(&sm.grad[256 * C], &maps.grad, binZ0 * C + 8 * C, binY0, xr, &sm.bar);
        tma_load_3d(&sm.pts[0], &maps.pts, binZ0 * 3, binY0, (p.d.pts_shared ? 0 : sample * H) + binX0, &sm.bar);
        if (PROB) tma_load_3d(&sm.aux[0], &maps.aux, binZ0 * 4, binY0, xr, &sm.bar);
    }

    // ---- candidates: the ascending list of this bin's supertile ------------------------------------------------
    const SplatWorkspace &ws = p.fwd;
    const bool slot_stores = DET && *p.canon != 0;   // cleared by the slot plan on overflow (or already by a stray point)
    const int s = supertile_of(ws, binX0, binY0);
    const int ncand = ws.counts[s];
    if (ncand == 0) {
        // No Gaussian to walk, but the point order is still this bin's to check: a point stored here may lie in a
        // covered voxel (several points in one voxel).  Waiting also keeps the CTA from exiting with its copies in flight.
        check_bin_order<C, PROB>(p, sm, binX0, binY0, binZ0);
        return;
    }
    bool tiles_ready = false;

    int cpos = 0;
    while (cpos < ncand) {
        __syncthreads();   // previous segment fully consumed
        if (tid == 0) sm.next = 0;   // published by the barriers of Phase A
        if (tid <= kVolKeys) sm.hist[tid] = 0;
        // ======================= Phase A: ordered survivors of the box test ==========================
        const int nlist = resolve_bin_list<NT, 2, kBinSeg>(p.d, ws, s, ncand, cpos, binX0, binY0, binZ0, sm.list, sm.warp_count);
        // ---- order the entries by clipped-box volume (counting sort; the order of the sum does not matter here) ----
        int mykey[kBinSeg / NT];
#pragma unroll
        for (int r = 0; r < kBinSeg / NT; ++r) {
            const int i = tid + r * NT;
            mykey[r] = 0;
            if (i < nlist) {
                const uint32_t m = sm.list[i].x;
                const int vol = __popc(m & 0xffu) * __popc((m >> 8) & 0xfu) * __popc(m >> 16);
                mykey[r] = (vol + 7) >> 3;
                atomicAdd(&sm.hist[mykey[r]], 1);
            }
        }
        __syncthreads();
        if (warp == 0) {   // exclusive prefix over the keys: lane L owns keys 2L+1, 2L+2 (key 0 is unused)
            const int c0 = sm.hist[2 * lane + 1], c1 = sm.hist[2 * lane + 2];
            int incl = c0 + c1;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            const int base = incl - c0 - c1;
            sm.hist[2 * lane + 1] = base;
            sm.hist[2 * lane + 2] = base + c0;
            // first entry of the wide class: keys >= kWideVol / 8
            constexpr int kWideKey = kWideVol / 8;
            if (2 * lane + 1 == kWideKey) sm.n_narrow = base;
            if (2 * lane + 2 == kWideKey) sm.n_narrow = base + c0;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < kBinSeg / NT; ++r) {
            const int i = tid + r * NT;
            if (i < nlist) sm.sorted[atomicAdd(&sm.hist[mykey[r]], 1)] = sm.list[i];
        }
        if (!tiles_ready) {   // the tiles were in flight during the first Phase A
            check_bin_order<C, PROB>(p, sm, binX0, binY0, binZ0);
            tiles_ready = true;
        }
        __syncthreads();

        // ======================= Phase B: eight lanes (or a whole warp) per listed Gaussian ===========
        const int n_narrow = sm.n_narrow, narrow_tickets = (n_narrow + 3) >> 2;
        const int tickets = narrow_tickets + (nlist - n_narrow);
#pragma unroll 1
        while (true) {
            int ticket = 0;
            if (lane == 0) ticket = atomicAdd(&sm.next, 1);
            ticket = __shfl_sync(0xffffffffu, ticket, 0);
            if (ticket >= tickets) break;
            const bool wide = ticket >= narrow_tickets;     // warp-uniform
            const int grp = lane >> 3, sub = lane & 7;
            const int e = wide ? n_narrow + (ticket - narrow_tickets) : 4 * ticket + grp;
            const bool have = wide || e < n_narrow;
            const uint2 ent = have ? sm.sorted[e] : make_uint2(0u, 0u);
            const int g = static_cast<int>(ent.y);
            const uint32_t xm = ent.x & 0xffu, ym = (ent.x >> 8) & 0xfu, zm = ent.x >> 16;
            const int x0 = __ffs(xm) - 1, nx = __popc(xm), y0 = __ffs(ym) - 1, ny = __popc(ym), z0 = __ffs(zm) - 1, nz = __popc(zm);
            const int vol = nx * ny * nz;   // 0 for a lane group without an entry
            GaussAcc<C, PROB> acc;
            acc.load_record(reinterpret_cast<const float4 *>(ws.records + static_cast<size_t>(g) * rec_floats(C)));
            // My lanes stride over the clipped box, z fastest; the stride is decomposed once into box steps.  A whole-warp
            // entry walks the two z halves of the box one after the other: the halves of the gradient tile are two TMA
            // boxes whose distance is a multiple of 128 bytes, so lanes on the same column and z & 7 of different halves
            // would hit the same banks (ncu: 39 % of the shared wavefronts of the prob config were such replays), while
            // neighbouring columns of ONE half sit 16 banks apart.
            const int first = wide ? lane : sub, stride = wide ? 32 : 8;
            const int nseg = wide ? 2 : 1;
#pragma unroll 1
            for (int sg = 0; sg < nseg; ++sg) {
                int zs = z0, nzh = nz;
                if (wide) {
                    zs = sg == 0 ? z0 : max(z0, 8);
                    nzh = sg == 0 ? min(z0 + nz, 8) - z0 : z0 + nz - zs;
                    if (nzh <= 0) continue;
                }
                const int volh = nx * ny * nzh;
                int t = small_div(first, nzh);
                int iz = first - t * nzh, ix = small_div(t, ny), iy = t - ix * ny;
                const int t2 = small_div(stride, nzh), sz = stride - t2 * nzh, sx = small_div(t2, ny), sy = t2 - sx * ny;
#pragma unroll 1
                for (int idx = first; idx < volh; idx += stride) {
                    const int col = (x0 + ix) * kBinY + (y0 + iy), Z = zs + iz;
                    PairData<C, PROB> pd;
                    pd.ok = true;
                    pd.shift = false;
                    const float *pp = &sm.pts[col * (kBinZ * 3) + Z * 3];
                    pd.px = pp[0]; pd.py = pp[1]; pd.pz = pp[2];
                    const float *row = &sm.grad[(Z >> 3) * (256 * C) + (col * 8 + (Z & 7)) * C];
                    if constexpr ((C & 1) == 0) {   // rows start 8-byte aligned
#pragma unroll
                        for (int k = 0; k < CP2; ++k) {
                            const float2 v = *reinterpret_cast<const float2 *>(row + 2 * k);
                            if (k & 1) { pd.raw[k >> 1].z = v.x; pd.raw[k >> 1].w = v.y; } else { pd.raw[k >> 1].x = v.x; pd.raw[k >> 1].y = v.y; }
                        }
                    } else {
#pragma unroll
                        for (int k = 0; k < CP2; ++k) {
                            const float a = row[2 * k], b = (2 * k + 1 < C) ? row[2 * k + 1] : 0.f;
                            if (k & 1) { pd.raw[k >> 1].z = a; pd.raw[k >> 1].w = b; } else { pd.raw[k >> 1].x = a; pd.raw[k >> 1].y = b; }
                        }
                    }
                    if (PROB) pd.ax = sm.aux[col * kBinZ + Z];
                    acc.template consume<false>(pd);
                    iz += sz;
                    const int cz = iz >= nzh;
                    iz -= cz ? nzh : 0;
                    iy += sy + cz;
                    const int cy = iy >= ny;
                    iy -= cy ? ny : 0;
                    ix += sx + cy;
                }
            }
            __syncwarp();
            float x[32];
            acc.to_vector(x);
            group8_transpose_reduce(x, lane);
            if (wide) {   // the four lane groups worked on the same Gaussian
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    x[i] += __shfl_xor_sync(0xffffffffu, x[i], 8);
                    x[i] += __shfl_xor_sync(0xffffffffu, x[i], 16);
                }
            }
            if (DET) {
                if (have && (!wide || grp == 0) && slot_stores) {
                    // slot of (g, this bin): slot_off[g] + the bin's position in the rectangle of bins g's box covers
                    const BoxBins bb(ws.boxes[g]);
                    const int rx = binX0 / kBinX - bb.b0[0], ry = binY0 / kBinY - bb.b0[1], rz = binZ0 / kBinZ - bb.b0[2];
                    const uint32_t slot = p.slot_off[g] + static_cast<uint32_t>((rx * bb.nb[1] + ry) * bb.nb[2] + rz);
                    float4 *row = reinterpret_cast<float4 *>(p.slots + static_cast<size_t>(slot) * 32);
                    row[sub] = make_float4(x[0], x[1], x[2], x[3]);   // values 4*sub .. 4*sub+3 (see group8_transpose_reduce)
                }
            } else if (have && (!wide || grp == 0)) {
                const int v0 = ((sub & 4) ? 16 : 0) + ((sub & 2) ? 8 : 0) + ((sub & 1) ? 4 : 0);
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (v0 + i < GaussAcc<C, PROB>::kVals) atomicAdd(p.sums + static_cast<size_t>(v0 + i) * p.d.G + g, x[i]);
            }
        }
    }
}

template <int C, bool PROB>
__global__ void __launch_bounds__(kBinThreads, 2) backward_bin_kernel(const BwdParams pb, int nbx,
                                                                       const __grid_constant__ BinMaps maps) {
    backward_bin<C, PROB, false>(pb, nbx, maps);
}

template <int C, bool PROB>
__global__ void __launch_bounds__(kBinThreads, 2) backward_bin_slots_kernel(const BwdParams pb, int nbx,
                                                                             const __grid_constant__ BinMaps maps) {
    backward_bin<C, PROB, true>(pb, nbx, maps);
}

// Deterministic mode, after list_kernel: per sample (one CTA), slot_off[g] = the exclusive prefix over g of the number of
// bins g's box covers, and the route word: bin route if the total fits the budget, else slot overflow -- which also
// clears the canon flag, so the bin kernel stores nothing and the Gaussian-centric chain produces the gradients (the
// hand-over a stray point triggers).
__global__ void __launch_bounds__(1024) slot_plan_kernel(const BwdParams pb) {
    pdl_launch_dependents();
    pdl_wait();   // the boxes of the pack kernel (list_kernel waited for it)
    const BwdParams p = sample_bwd(pb, blockIdx.x);
    const unsigned long long total = cta_ordered_scan<1024>(
        p.d.G, [&](int g) { return static_cast<unsigned long long>(BoxBins(p.fwd.boxes[g]).count()); },
        [&](int g, unsigned long long o) { p.slot_off[g] = static_cast<uint32_t>(o); });
    if (threadIdx.x == 0) {
        const bool fits = total <= static_cast<unsigned long long>(p.budget);
        *route_word(p.canon) = fits ? kRouteBin : kRouteSlotOverflow;
        if (!fits) *p.canon = 0;
    }
}

__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

constexpr int kWarpSlots = 128;   // Gaussians with more slot rows are summed by the whole CTA

// Deterministic mode: one warp per Gaussian sums its slot rows and finish() (splat_bwd_common.cuh) writes the gradients.
// Lane l adds float4 l & 7 of rows l >> 3, (l >> 3) + 4, ... in ascending order, then a fixed butterfly over the four
// row columns; a Gaussian with more than kWarpSlots rows (the whole-grid one covers every bin) is summed the same way by
// all 256 threads (32 row columns) with a fixed tree over the warps.  The order depends on the row count only.
template <int C, bool PROB>
__global__ void __launch_bounds__(256) bin_slot_finish_kernel(const BwdParams pb) {
    pdl_launch_dependents();
    pdl_wait();
    const BwdParams p = sample_bwd(pb, blockIdx.y);
    const bool canon = *p.canon != 0;
    if (blockIdx.x == 0 && threadIdx.x == 0 && !canon && *route_word(p.canon) == kRouteBin) *route_word(p.canon) = kRouteStrayPoints;
    if (!canon) return;
    const int G = p.d.G, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, q = lane & 7;
    const PackedBox *boxes = p.fwd.boxes;
    const uint32_t *off = p.slot_off;
    const float4 *rows = reinterpret_cast<const float4 *>(p.slots);
    __shared__ int s_wide[8];
    __shared__ float4 s_red[8][8];
    // lane l ends up with value l of the total of quads t (lane j holds quad j & 7)
    auto value_of = [&](float4 t) {
        const int src = lane >> 2;
        const float a = __shfl_sync(0xffffffffu, t.x, src), b = __shfl_sync(0xffffffffu, t.y, src);
        const float c = __shfl_sync(0xffffffffu, t.z, src), d = __shfl_sync(0xffffffffu, t.w, src);
        const int k = lane & 3;
        return k == 0 ? a : (k == 1 ? b : (k == 2 ? c : d));
    };
    const int g = blockIdx.x * 8 + warp;
    int n = 0;
    size_t o = 0;
    if (g < G) {
        n = BoxBins(boxes[g]).count();
        o = off[g];
    }
    const bool wide = n > kWarpSlots;
    if (g < G && !wide) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s = lane >> 3; s < n; s += 4) a = add4(a, rows[(o + s) * 8 + q]);
        a = add4(a, make_float4(__shfl_xor_sync(0xffffffffu, a.x, 8), __shfl_xor_sync(0xffffffffu, a.y, 8),
                                __shfl_xor_sync(0xffffffffu, a.z, 8), __shfl_xor_sync(0xffffffffu, a.w, 8)));
        a = add4(a, make_float4(__shfl_xor_sync(0xffffffffu, a.x, 16), __shfl_xor_sync(0xffffffffu, a.y, 16),
                                __shfl_xor_sync(0xffffffffu, a.z, 16), __shfl_xor_sync(0xffffffffu, a.w, 16)));
        finish<C, PROB>(p, g, value_of(a), lane, false);
    }
    if (lane == 0) s_wide[warp] = g < G && wide;
    __syncthreads();
    for (int w = 0; w < 8; ++w) {
        if (!s_wide[w]) continue;   // CTA-uniform
        const int gw = blockIdx.x * 8 + w;
        const int nw = BoxBins(boxes[gw]).count();
        const size_t ow = off[gw];
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s = threadIdx.x >> 3; s < nw; s += 32) a = add4(a, rows[(ow + s) * 8 + q]);
        a = add4(a, make_float4(__shfl_xor_sync(0xffffffffu, a.x, 8), __shfl_xor_sync(0xffffffffu, a.y, 8),
                                __shfl_xor_sync(0xffffffffu, a.z, 8), __shfl_xor_sync(0xffffffffu, a.w, 8)));
        a = add4(a, make_float4(__shfl_xor_sync(0xffffffffu, a.x, 16), __shfl_xor_sync(0xffffffffu, a.y, 16),
                                __shfl_xor_sync(0xffffffffu, a.z, 16), __shfl_xor_sync(0xffffffffu, a.w, 16)));
        if (lane < 8) s_red[warp][lane] = a;
        __syncthreads();
        if (warp == 0) {
            float4 t = add4(add4(add4(s_red[0][q], s_red[1][q]), add4(s_red[2][q], s_red[3][q])),
                            add4(add4(s_red[4][q], s_red[5][q]), add4(s_red[6][q], s_red[7][q])));
            finish<C, PROB>(p, gw, value_of(t), lane, false);
        }
        __syncthreads();
    }
}

// One thread per Gaussian: the raw sums of all bins ([32][G], value-major: coalesced reads) -> the gradients, i.e. the
// per-Gaussian linear maps of finish() (splat_bwd_common.cuh): d(mean) = -A * sum(w d), d(cov) = -(1/2 | 1) * sum(w d d^T)
// (+ the determinant terms of the prob variant), d(sem) = opacity * sum(E g) for the base variant.
template <int C, bool PROB>
__global__ void __launch_bounds__(128) bin_finish_kernel(const BwdParams pb) {
    pdl_launch_dependents();
    pdl_wait();
    const BwdParams p = sample_bwd(pb, blockIdx.y);
    if (*p.canon == 0) return;
    const int g = blockIdx.x * 128 + threadIdx.x;
    const int G = p.d.G;
    if (g >= G) return;
    const float *sums = p.sums + g;
    float v[32];
#pragma unroll
    for (int i = 0; i < GaussAcc<C, PROB>::kVals; ++i) v[i] = __ldg(sums + static_cast<size_t>(i) * G);
    float c6[6];
    load_cov6_in(p.d, p.in, g, c6);
    const float a = c6[0], b = c6[1], c = c6[2], d = c6[3], e = c6[4], f = c6[5];
    p.gr.means_grad[3 * g + 0] = -(a * v[0] + d * v[1] + f * v[2]);
    p.gr.means_grad[3 * g + 1] = -(d * v[0] + b * v[1] + e * v[2]);
    p.gr.means_grad[3 * g + 2] = -(f * v[0] + e * v[1] + c * v[2]);
    p.gr.opacity_grad[g] = v[3];
    float gc[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) gc[i] = (i < 3) ? -0.5f * v[4 + i] : -v[4 + i];
    if (PROB) {
        const float sg = v[10 + C];
        const float m[6] = {b * c - e * e, a * c - f * f, a * b - d * d, 2.f * (e * f - c * d), 2.f * (d * f - a * e), 2.f * (d * e - b * f)};
#pragma unroll
        for (int i = 0; i < 6; ++i) gc[i] = fmaf(sg, m[i], gc[i]);
    }
    if (p.d.cov_stride == 9) {   // the six gathered entries [0,4,8,1,5,2] of the 3x3 carry the gradient, the lower triangle gets 0
        float *o = p.gr.cov_grad + 9 * static_cast<size_t>(g);
        o[0] = gc[0]; o[1] = gc[3]; o[2] = gc[5]; o[3] = 0.f; o[4] = gc[1]; o[5] = gc[4]; o[6] = 0.f; o[7] = 0.f; o[8] = gc[2];
    } else {
        float *o = p.gr.cov_grad + 6 * static_cast<size_t>(g);
#pragma unroll
        for (int i = 0; i < 6; ++i) o[i] = gc[i];
    }
    const float scale = PROB ? 1.f : p.in.opacities[g];
#pragma unroll
    for (int k = 0; k < C; ++k) p.gr.semantics_grad[static_cast<size_t>(g) * C + k] = scale * v[10 + k];
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = [] {
        void *f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            f = nullptr;
        return reinterpret_cast<EncodeTiledFn>(f);
    }();
    return fn;
}

// fp32 tensor [rows][W][inner] (contiguous) with boxes {box_inner, 4, 8}
static bool make_map(CUtensorMap *m, const void *base, long long rows, int W, int inner, int box_inner) {
    EncodeTiledFn fn = encode_tiled();
    if (!fn) return false;
    const cuuint64_t dims[3] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(rows)};
    const cuuint64_t strides[2] = {static_cast<cuuint64_t>(inner) * 4, static_cast<cuuint64_t>(inner) * 4 * W};
    const cuuint32_t box[3] = {static_cast<cuuint32_t>(box_inner), kBinY, kBinX};
    const cuuint32_t estr[3] = {1, 1, 1};
    return fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Can the bin-centric kernel serve this call (if the points turn out to be in canonical order on the device)?
bool backward_bin_eligible(const gf_splat_desc &d, const gf_splat_inputs &in, const gf_splat_grads &gr) {
    if (encode_tiled() == nullptr) return false;
    if (static_cast<long long>(d.N) != static_cast<long long>(d.H) * d.W * d.D || d.N == 0 || d.G == 0) return false;
    if ((d.D & 3) != 0 || 8 * d.C > 256) return false;   // 16-byte strides of the tensor maps, box <= 256 elements
    auto al16 = [](const void *q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
    return al16(in.pts) && al16(gr.logits_grad);
}

template <int C, bool PROB>
static int launch_bin_t(const BwdParams &bp, bool det, const BinMaps &maps, cudaStream_t stream) {
    const gf_splat_desc &d = bp.d;
    const int B = batch_of(d);
    const int nzc = (d.D + kBinZ - 1) / kBinZ, nby = (d.W + kBinY - 1) / kBinY, nbx = (d.H + kBinX - 1) / kBinX;
    GF_REQUIRE(nby <= 65535 && static_cast<long long>(nbx) * B <= 65535, GF_ERR_UNSUPPORTED,
               "splat backward: grid x batch too large for the bin launch");
    const size_t smem = sizeof(BinSmem<C, PROB>);
    if (det) {
        GF_CUDA_TRY(launch_chained(slot_plan_kernel, dim3(B), dim3(1024), 0, stream, bp));
        GF_CUDA_TRY(cudaFuncSetAttribute(backward_bin_slots_kernel<C, PROB>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        GF_CUDA_TRY(launch_chained(backward_bin_slots_kernel<C, PROB>, dim3(nzc, nby, nbx * B), dim3(kBinThreads), smem, stream, bp, nbx, maps));
        GF_CUDA_TRY(launch_chained(bin_slot_finish_kernel<C, PROB>, dim3((d.G + 7) / 8, B), dim3(256), 0, stream, bp));
        return GF_OK;
    }
    // per call: the attribute is per device, and a process may drive several
    GF_CUDA_TRY(cudaFuncSetAttribute(backward_bin_kernel<C, PROB>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    GF_CUDA_TRY(launch_chained(backward_bin_kernel<C, PROB>, dim3(nzc, nby, nbx * B), dim3(kBinThreads), smem, stream, bp, nbx, maps));
    GF_CUDA_TRY(launch_chained(bin_finish_kernel<C, PROB>, dim3((d.G + 127) / 128, B), dim3(128), 0, stream, bp));
    return GF_OK;
}

// bp: the launch parameters of the backward (batch-level pointers), with the supertile lists built for this call
int launch_backward_bin(const BwdParams &bp, bool det, cudaStream_t stream) {
    const gf_splat_desc &d = bp.d;
    const long long B = batch_of(d);
    BinMaps maps;
    bool ok = make_map(&maps.grad, bp.gr.logits_grad, B * d.H, d.W, d.D * d.C, 8 * d.C);
    ok = ok && make_map(&maps.pts, bp.in.pts, (d.pts_shared ? 1 : B) * d.H, d.W, d.D * 3, kBinZ * 3);
    if (d.variant == GF_SPLAT_PROB) ok = ok && make_map(&maps.aux, bp.aux, B * d.H, d.W, d.D * 4, kBinZ * 4);
    else maps.aux = maps.pts;
    GF_REQUIRE(ok, GF_ERR_CUDA, "splat backward: cuTensorMapEncodeTiled failed");
    const bool prob = d.variant == GF_SPLAT_PROB;
    return dispatch_classes(d.C, "splat backward", [&](auto cc) {
        constexpr int C = decltype(cc)::value;
        return prob ? launch_bin_t<C, true>(bp, det, maps, stream) : launch_bin_t<C, false>(bp, det, maps, stream);
    });
}

}  // namespace gf
