// The tile walker of the render kernel: a CTA owns a bin of 8 x 4 columns x 16 z; it resolves its own ordered
// Gaussian list from the supertile list (Phase A), streams the records through a shared-memory ring (Phase B)
// and lets every lane walk ITS OWN hits of a batch in ascending Gaussian order (lane-private traversal).
#pragma once
#include "splat_render.cuh"

namespace gf {

constexpr int kVoxT = 4;        // voxels per thread: a z quad
constexpr int kQuadSeg = 512;   // list entries resolved per segment
constexpr int kBatch = 32;      // records staged per ring slot; a lane keeps its hit mask of a batch in one word
// ring slots: a warp may run up to kRing-2 batches ahead of the slowest one
// (measured on a B200 before the H100 port: 5, 6, 7 slots 72.0 us per step, 4 and 8 slots 73.4 us)
constexpr int kRing = 5;

// Shared-memory row of a staged record: the 128-byte record followed by 16 bytes of padding, so that chunk c of row j
// starts at bank group (j + c) mod 8 and lanes of one warp reading the same chunk of DIFFERENT records fall into
// different bank groups -- the effect of an XOR swizzle, but a chunk's address is row + 16*c, an immediate offset of the
// load (the XOR cost one LOP3 per chunk and step: 8 of 92 instructions).
template <int C>
struct RenderSmem {
    static constexpr int REC = rec_floats(C);
    static constexpr int ROW = REC + 4;        // floats per staged row
    static constexpr int NT = kRenderThreads;
    // Epilogue tile: the CTA's logits in [N, C] order, one row of kBinZ voxels per column (x-major), each row padded
    // by 16 bytes so that the two z quads of neighbouring lanes fall into different bank groups.  A row is one
    // contiguous run of the output when D % kBinZ == 0, copied out with one bulk copy.
    static constexpr int TILE_ROW = kBinZ * C + 4;
    struct Walk {
        alignas(128) float stage[kRing][kBatch * ROW];
        alignas(8) uint2 list[kQuadSeg + kBatch];  // x: box relative to the bin as bit masks, y: Gaussian index
        uint32_t hitw[kQuadSeg / kBatch + 1][16];  // per batch: bit j of word i = entry j covers x position i (0..7), y position i-8 (8..11), z quad i-12 (12..15)
    };
    union {
        Walk w;                                              // Phase A and B
        alignas(128) float tile[kBinX * kBinY][TILE_ROW];    // epilogue: the walk's buffers are dead by then
    };
    alignas(8) uint64_t bar_full[kRing];       // records of the slot have landed (one cp.async arrival per thread)
    alignas(8) uint64_t bar_empty[kRing];      // every warp is done with the slot (one arrival per warp)
    int warp_count[2][NT / 32];
    float ce[NT / 32][2];                      // per-warp cross-entropy partials of the epilogue
    uint32_t stray_warp[NT / 32];              // per warp: some lane has a point outside canonical voxel order
#ifdef GF_RENDER_TIMING
    unsigned long long t_phase[8];             // cycle sums: prologue, Phase A, Phase B, epilogue (thread 0); all warps: wait-full, wait-empty + issue, hit masks, walk
#endif
};

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
// the mbarrier receives one arrival from this thread when all its earlier cp.async have landed
__device__ __forceinline__ void cp_async_arrive_on(uint64_t *bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_one(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void st_shared16(void *smem_dst, float4 v) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(smem_u32(smem_dst)), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}
// this thread's shared-memory writes become visible to the bulk copies (async proxy) issued after the next barrier
__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// bulk copy of `bytes` (a multiple of 16, both addresses 16-byte aligned) from shared to global memory
__device__ __forceinline__ void bulk_copy_s2g(void *gmem_dst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}
// commit this thread's bulk copies and wait until they have READ their shared-memory sources; the global writes drain
// on their own and are visible to later kernels of the stream
__device__ __forceinline__ void bulk_commit_wait_read() {
    asm volatile("cp.async.bulk.commit_group;\n\tcp.async.bulk.wait_group.read 0;" ::: "memory");
}

// One staged record as a lane sees it: `addr` is the shared-space address of its row, chunk i sits 16*i bytes further.
struct RecView {
    uint32_t addr;
    __device__ __forceinline__ float4 chunk(int i) const {
        float4 v;
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr + 16u * static_cast<uint32_t>(i)));
        return v;
    }
};

// The caller supplies one callable:
//   step(RecView record, uint32_t zbits, bool active)   evaluate + accumulate one (record, my z quad) pair; `active`
//       says whether this lane has a record in this step, bit v of zbits whether its voxel v lies inside the box.
//       Inactive lanes must not touch `record`.
//
// Lane-private traversal: a Gaussian's box covers only part of a warp's 4 x 4 x 8 footprint (17.7 of 32 lanes on the
// nuScenes workload), so marching all lanes through every record that touches the footprint leaves almost half of them
// idle in every step.  Instead each lane gets the bit mask of the records of the batch that cover ITS column and z
// quad -- the box masks are separable, so 16 ballots per batch and CTA (8 x bits, 4 y bits, 4 z quads; three word loads
// and two ANDs per lane) produce all 128 masks -- and walks its own bits in ascending order (the reference's summation order per voxel); the warp iterates
// max-over-lanes popcount times instead of once per touching record.
// Two step functors: `step_fast` is used when `fast` (CTA-uniform) says every thread qualifies for it, `step` otherwise;
// only the innermost loop exists twice.
template <int C, class StepFast, class Step>
__device__ __forceinline__ void walk_tile(const RenderParams &p, RenderSmem<C> &sm, int binX0, int binY0, int binZ0,
                                          int my_zshift, bool fast, StepFast &&step_fast, Step &&step) {
    constexpr int REC = rec_floats(C), ROW = RenderSmem<C>::ROW;
    constexpr int NT = kRenderThreads, NWARP = NT / 32, VOX = kVoxT;
    constexpr uint32_t VMASK = (1u << VOX) - 1u;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
#pragma unroll
        for (int r = 0; r < kRing; ++r) {
            mbar_init(&sm.bar_full[r], NT);
            mbar_init(&sm.bar_empty[r], NWARP);
        }
        mbar_fence_init();
    }
    uint32_t gb = 0;   // batches consumed so far by this CTA: drives ring slots and barrier parities
    // (the __syncthreads of Phase A below publishes the barrier initialisation)

    // ---- candidates: the ascending list of this bin's supertile ------------------------------------
    const int s = supertile_of(p.ws, binX0, binY0);
    const int ncand = p.ws.counts[s];

    int cpos = 0;
    while (cpos < ncand) {
        __syncthreads();   // previous segment fully consumed (and, the first time, barriers initialised)
#ifdef GF_RENDER_TIMING
        const long long tA0 = clock64();
#endif
        // ======================= Phase A: ordered survivors of the box test ==========================
        const int nlist = resolve_bin_list<NT, 4, kQuadSeg>(p.d, p.ws, s, ncand, cpos, binX0, binY0, binZ0, sm.w.list, sm.warp_count);
        // pad the last batch with empty entries (all-zero masks, so nobody visits them)
        if (tid < kBatch && nlist + tid < ((nlist + kBatch - 1) / kBatch) * kBatch) sm.w.list[nlist + tid] = make_uint2(0u, 0u);
        __syncthreads();
        const int nchunks = (nlist + kBatch - 1) / kBatch;
        auto issue = [&](int k, uint32_t b_index) {  // batch k of this segment -> ring slot b_index % kRing
            const int slot = b_index % kRing;
            const uint32_t use = b_index / kRing;
            if (use > 0) mbar_wait(&sm.bar_empty[slot], (use - 1) & 1);   // previous occupant released by all warps
#pragma unroll
            for (int q = 0; q < (kBatch * 8 + NT - 1) / NT; ++q) {     // 32 records x 8 x 16 B = 256 copies
                const int piece = tid + NT * q, row = piece >> 3, col = (piece & 7) * 4;
                if (piece < kBatch * 8 && k * kBatch + row < nlist) {
                    const uint32_t g = sm.w.list[k * kBatch + row].y;
                    cp_async16(&sm.w.stage[slot][row * ROW + col], p.ws.records + static_cast<size_t>(g) * REC + col);
                }
            }
            cp_async_arrive_on(&sm.bar_full[slot]);
        };
#pragma unroll 1
        for (int k = 0; k < kRing - 1 && k < nchunks; ++k) issue(k, gb + k);
        // The box masks are separable, so 16 ballots per batch -- taken ONCE per CTA, the batches dealt to the four warps --
        // transpose them into 16 words (which entries cover x position i / y position i / z quad i); a lane's hit mask of a
        // batch is then the AND of three of those words (ten ballots per warp and batch before: 9 % of Phase B).
        for (int b = warp; b < (nlist + kBatch - 1) / kBatch; b += NWARP) {
            const uint32_t ex = sm.w.list[b * kBatch + lane].x;
            uint32_t mine = 0u;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const bool covers = i < 12 ? ((ex >> i) & 1u) != 0u : ((ex >> (16 + VOX * (i - 12))) & VMASK) != 0u;
                const uint32_t w = __ballot_sync(0xffffffffu, covers);
                if (lane == i) mine = w;
            }
            if (lane < 16) sm.w.hitw[b][lane] = mine;
        }
        __syncthreads();
#ifdef GF_RENDER_TIMING
        const long long tB0 = clock64();
        if (tid == 0) sm.t_phase[1] += static_cast<unsigned long long>(tB0 - tA0);
#endif

        // ======================= Phase B: stream records and accumulate ==============================
        // No CTA-wide barrier in this loop: full[] / empty[] mbarriers let the four warps drift apart by
        // up to kRing-2 batches, so a warp whose footprint is touched by few records does not wait.
#pragma unroll 1
        for (int k = 0; k < nchunks; ++k, ++gb) {
#ifdef GF_RENDER_TIMING
            const long long tk0 = clock64();
#endif
            const int slot = gb % kRing;
            const uint32_t stage_base = smem_u32(&sm.w.stage[slot][0]);
            // bit j of `hits`: record j of this batch covers my column and my z quad (padded entries are all-zero)
            uint32_t hits;
            {
                const uint32_t *hw = sm.w.hitw[k];
                hits = hw[4 * (warp & 1) + (lane >> 3)] & hw[8 + ((lane >> 1) & 3)] & hw[12 + 2 * (warp >> 1) + (lane & 1)];
            }
#ifdef GF_RENDER_TIMING
            const long long tw0 = clock64();
#endif
            mbar_wait(&sm.bar_full[slot], (gb / kRing) & 1);
#ifdef GF_RENDER_TIMING
            const long long tw1 = clock64();
#endif
            // the warp takes as many steps as its busiest lane has hits in this batch
            const int nsteps = __reduce_max_sync(0xffffffffu, __popc(hits));
            auto pop = [&](bool &act, RecView &rv, uint32_t &zb) {
                act = hits != 0;
                const int jraw = __ffs(static_cast<int>(hits)) - 1;          // my lowest remaining hit; -1 when I have none
                hits &= hits - 1;                                             // 0 stays 0
                rv.addr = stage_base + static_cast<uint32_t>(jraw * (ROW * 4));   // an inactive lane never dereferences it
                const uint32_t e = sm.w.list[k * kBatch + (act ? jraw : 0)].x;
                zb = (e >> my_zshift) & VMASK;
            };
            if (fast) {
#pragma unroll 2
                for (int st = 0; st < nsteps; ++st) {
                    bool act; RecView rv; uint32_t zb;
                    pop(act, rv, zb);
                    step_fast(rv, zb, act);
                }
            } else {
#pragma unroll 2
                for (int st = 0; st < nsteps; ++st) {
                    bool act; RecView rv; uint32_t zb;
                    pop(act, rv, zb);
                    step(rv, zb, act);
                }
            }
            __syncwarp();
#ifdef GF_RENDER_TIMING
            const long long tw2 = clock64();
#endif
            if (lane == 0) mbar_arrive_one(&sm.bar_empty[slot]);       // my warp is done with this slot
            if (k + kRing - 1 < nchunks) issue(k + kRing - 1, gb + kRing - 1);
#ifdef GF_RENDER_TIMING
            if (lane == 0) {
                atomicAdd(&sm.t_phase[4], static_cast<unsigned long long>(tw1 - tw0));
                atomicAdd(&sm.t_phase[5], static_cast<unsigned long long>(clock64() - tw2));
                atomicAdd(&sm.t_phase[6], static_cast<unsigned long long>(tw0 - tk0));
                atomicAdd(&sm.t_phase[7], static_cast<unsigned long long>(tw2 - tw1));
            }
#endif
        }
#ifdef GF_RENDER_TIMING
        if (tid == 0) sm.t_phase[2] += static_cast<unsigned long long>(clock64() - tB0);
#endif
    }
}

}  // namespace gf
