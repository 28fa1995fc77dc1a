// Splat stage 2 — the render kernels (replaces FORWARD::renderCUDA, model/head/localagg/src/forward.cu:35-82
// and the prob variant model/head/localagg_prob/src/forward.cu:35-102).
//
// render_tile_kernel    the default tile kernel for points in canonical voxel order (see its header
//                       comment below); stray points are detected per voxel and re-evaluated exactly.
// render_points_kernel  arbitrary points (N != H*W*D, several per voxel): one thread per point walks
//                       the supertile list with the exact box test.
#include "splat_host.cuh"
#include "splat_tile.cuh"

namespace gf {

// SIMT render kernel: bin = 8 x 4 columns x 16 z, 4 consecutive z voxels per thread with 4 x C accumulators in
// registers (36 packed fp32 pairs); a warp covers 4 x 4 columns x 8 z.  128 threads, 128 registers, 4 CTAs per SM.
//   * Phase A resolves the bin's ordered Gaussian list; each entry carries the box clipped to the bin
//     as bit masks (x: 8 bits, y: 4 bits, z: 16 bits), so Phase B never unpacks coordinates.
//   * Phase B streams the records (cp.async into an mbarrier-guarded ring); every lane walks the records that cover
//     its own column and z quad (splat_tile.cuh), and the class accumulation runs on packed fp32 pairs (FFMA2).
//   * The epilogue writes the logits ([N,C] and / or class-major [C,N]), the fused arg-max and, on request, the
//     softmax cross-entropy partial sums of the CTA's voxels.
// blockIdx = (z chunk, bin y, sample * nbx + bin x): one grid covers the whole batch.
template <int C, bool PROB>
__global__ void __launch_bounds__(kRenderThreads, PROB ? 3 : 4) render_tile_kernel(const RenderParams pb) {
    constexpr int REC = rec_floats(C);
    constexpr int CP2 = (C + 1) / 2;   // packed class pairs
    constexpr int VOX = kVoxT;
    static_assert(REC == 32, "one record = 128 bytes");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    RenderSmem<C> &sm = *reinterpret_cast<RenderSmem<C> *>(smem_raw);
#ifdef GF_RENDER_TIMING
    const long long t_start = clock64();
    if (threadIdx.x < 8) sm.t_phase[threadIdx.x] = 0ull;
#endif
    const int sample = blockIdx.z / pb.nbx;
    const RenderParams pin = sample_params(pb, sample);   // inputs + workspace of my sample; outputs: see the epilogue

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int H = pin.d.H, W = pin.d.W, D = pin.d.D;

    // ---- which voxels are mine -------------------------------------------------------------------
    const int binX0 = (blockIdx.z - sample * pb.nbx) * kBinX, binY0 = blockIdx.y * kBinY, binZ0 = blockIdx.x * kBinZ;
    const int lx = (warp & 1) * 4 + (lane >> 3), ly = (lane >> 1) & 3, lq = (warp >> 1) * 2 + (lane & 1);  // z quad
    const int X = binX0 + lx, Y = binY0 + ly, Z0 = binZ0 + VOX * lq;
    const bool col_ok = X < H && Y < W;
    const bool live = col_ok && Z0 < D;
    const long long n0 = (static_cast<long long>(X) * W + Y) * D + Z0;
    const bool vec_ok = pin.vec_ok != 0;  // D % 4 == 0 (then n0 % 4 == 0 and Z0+3 < D whenever Z0 < D) and aligned tensors

    float px[VOX], py[VOX], pz[VOX];
    bool vox_ok[VOX];
#pragma unroll
    for (int v = 0; v < VOX; ++v) {
        vox_ok[v] = col_ok && (Z0 + v) < D;
        px[v] = py[v] = pz[v] = 0.f;
    }
    uint32_t stray = 0;   // bit v: point n0+v does not sit in voxel n0+v
    if (live) {
        if (vec_ok) {
            // 12 contiguous floats, 16-byte aligned (n0 % 4 == 0 and an aligned tensor, see launch_render)
            float raw[3 * VOX];
            const float4 *src = reinterpret_cast<const float4 *>(pin.pts + 3 * n0);
#pragma unroll
            for (int i = 0; i < 3 * VOX / 4; ++i) {
                const float4 t = __ldg(src + i);
                raw[4 * i] = t.x; raw[4 * i + 1] = t.y; raw[4 * i + 2] = t.z; raw[4 * i + 3] = t.w;
            }
#pragma unroll
            for (int v = 0; v < VOX; ++v) { px[v] = raw[3 * v]; py[v] = raw[3 * v + 1]; pz[v] = raw[3 * v + 2]; }
        } else {
#pragma unroll
            for (int v = 0; v < VOX; ++v)
                if (vox_ok[v]) {
                    px[v] = __ldg(pin.pts + 3 * (n0 + v));
                    py[v] = __ldg(pin.pts + 3 * (n0 + v) + 1);
                    pz[v] = __ldg(pin.pts + 3 * (n0 + v) + 2);
                }
        }
        // canonical-order check: point n must lie in voxel n.  A cheap reciprocal estimate settles every
        // point that is not within 1e-3 cells of a voxel face; only those pay the exact IEEE divisions.
        const float inv = __frcp_rn(pin.d.grid_size);
#pragma unroll
        for (int v = 0; v < VOX; ++v)
            if (vox_ok[v]) {
                int ix, iy, iz;
                if (pin.points_int) {
                    ix = pin.points_int[3 * (n0 + v)];
                    iy = pin.points_int[3 * (n0 + v) + 1];
                    iz = pin.points_int[3 * (n0 + v) + 2];
                } else {
                    const float fx = (px[v] - pin.d.pc_min[0]) * inv - static_cast<float>(X);
                    const float fy = (py[v] - pin.d.pc_min[1]) * inv - static_cast<float>(Y);
                    const float fz = (pz[v] - pin.d.pc_min[2]) * inv - static_cast<float>(Z0 + v);
                    const float lo_m = 1e-3f, hi_m = 1.f - 1e-3f;
                    if (fx > lo_m && fx < hi_m && fy > lo_m && fy < hi_m && fz > lo_m && fz < hi_m) {
                        ix = X; iy = Y; iz = Z0 + v;
                    } else {
                        ix = voxel_coord(px[v], pin.d.pc_min[0], pin.d.grid_size);
                        iy = voxel_coord(py[v], pin.d.pc_min[1], pin.d.grid_size);
                        iz = voxel_coord(pz[v], pin.d.pc_min[2], pin.d.grid_size);
                    }
                }
                if (!(ix == X && iy == Y && iz == Z0 + v)) stray |= 1u << v;
            }
    }
    // do my 4 points share x and y exactly?  (decided once; the branch on it is warp-uniform in practice)
    bool column = true;
#pragma unroll
    for (int v = 1; v < VOX; ++v) column = column && px[v] == px[0] && py[v] == py[0];
    const int my_zshift = 16 + VOX * lq;   // entry word: x mask [0,8) | y mask [8,12) | z mask [16,32)
    int my_zlevel = Z0;                     // first z level of my quad: shift of a record's z-level mask
    asm volatile("" : "+r"(my_zlevel));     // opaque: otherwise rebuilt from %tid / %ctaid in every step of the walk

    float2 acc[VOX][CP2];
    float zsum[VOX], dens[VOX], keep[VOX];
#pragma unroll
    for (int v = 0; v < VOX; ++v) {
#pragma unroll
        for (int c = 0; c < CP2; ++c) acc[v][c] = make_float2(0.f, 0.f);
        zsum[v] = 0.f; dens[v] = 0.f; keep[v] = 1.f;
    }

    // Everything above depends on the caller's inputs only; the records, boxes, lists and the status word
    // come from the two preparation kernels, which this grid may have been launched ahead of.
    pdl_wait();
    if (stray) atomicOr(pin.ws.flags, GF_FLAG_GENERIC_PATH);
    {
        const bool warp_stray = __any_sync(0xffffffffu, stray != 0);   // read by the epilogue; kept out of registers
        if (lane == 0) sm.stray_warp[warp] = warp_stray;
    }
#ifdef GF_RENDER_TIMING
    if (tid == 0) sm.t_phase[0] = static_cast<unsigned long long>(clock64() - t_start);
#endif
    // One step of a lane = one (record, my 4 voxels) evaluation: exponent and weights from the record's three geometry
    // chunks, then the class accumulation (4 x C/2 packed FMAs) with its class chunks read where they are used.
    static_assert(C >= 16 && C <= 20, "forward record layout: class pairs 0..7 are always present");
    auto accumulate = [&](const RecView rec, const float4 g2c, const float (&wv)[VOX]) {
        // forward record layout (common.cuh): class pairs 0..7 in chunks 3..6, pair 8 in the coefficient chunk, pair 9 in chunk 7
#pragma unroll
        for (int c4 = 0; c4 < 4; ++c4) {
            const float4 s4 = rec.chunk(3 + c4);
#pragma unroll
            for (int v = 0; v < VOX; ++v) {
                const float2 ww = make_float2(wv[v], wv[v]);
                acc[v][2 * c4] = ffma2(make_float2(s4.x, s4.y), ww, acc[v][2 * c4]);
                acc[v][2 * c4 + 1] = ffma2(make_float2(s4.z, s4.w), ww, acc[v][2 * c4 + 1]);
            }
        }
        if constexpr (CP2 > 8) {
#pragma unroll
            for (int v = 0; v < VOX; ++v) acc[v][8] = ffma2(make_float2(g2c.z, g2c.w), make_float2(wv[v], wv[v]), acc[v][8]);
        }
        if constexpr (CP2 > 9) {
            const float4 s4 = rec.chunk(7);
#pragma unroll
            for (int v = 0; v < VOX; ++v) acc[v][9] = ffma2(make_float2(s4.x, s4.y), make_float2(wv[v], wv[v]), acc[v][9]);
        }
    };
    // My 4 points share x and y (voxel centres of one z column -- every shipped config,
    // dataset/transform_3d.py:484-499 without perturbation): the exponent is a quadratic
    // in dz alone, q = (cc*dz + B)*dz + A, with A and B evaluated once per record; the per-voxel part runs on
    // packed fp32 pairs (voxels (0,1) and (2,3) share each instruction).
    auto step_column = [&](const RecView rec, uint32_t zb_entry, bool active) {
        if (!active) return;
        const float4 g0 = rec.chunk(0), g1 = rec.chunk(1), g2c = rec.chunk(2);
        // base variant: the record's amplitude slot holds the z levels of the clipped box as a bit mask (pack kernel; the
        // grid has at most 32 levels on this path, see `all_column`), so the list entry is not read at all
        const uint32_t zb = PROB ? zb_entry : (__float_as_uint(g0.w) >> my_zlevel) & ((1u << VOX) - 1u);
        float wv[VOX];
        const float dx = g0.x - px[0], dy = g0.y - py[0];
        float t1 = g1.x * dx;
        t1 = fmaf(g1.w, dy, t1);
        float A = t1 * dx;
        A = fmaf(g1.y * dy, dy, A);
        const float B = fmaf(g2c.x, dy, g2c.y * dx);
#pragma unroll
        for (int h2 = 0; h2 < VOX / 2; ++h2) {
            const int v0 = 2 * h2, v1 = v0 + 1;
            const float2 dz = fadd2(make_float2(g0.z, g0.z), make_float2(-pz[v0], -pz[v1]));
            float2 q = ffma2(make_float2(g1.z, g1.z), dz, make_float2(B, B));
            q = ffma2(q, dz, make_float2(A, A));
            const float E0 = ((zb >> v0) & 1u) ? ex2_approx(q.x) : 0.f;
            const float E1 = ((zb >> v1) & 1u) ? ex2_approx(q.y) : 0.f;
            wv[v0] = PROB ? g0.w * E0 : E0;      // base: the opacity is folded into the class vector (pack kernel)
            wv[v1] = PROB ? g0.w * E1 : E1;
            if (PROB) {
                zsum[v0] += wv[v0]; dens[v0] += E0; keep[v0] *= (1.f - E0);
                zsum[v1] += wv[v1]; dens[v1] += E1; keep[v1] *= (1.f - E1);
            }
        }
        accumulate(rec, g2c, wv);
    };
    // general points: the full quadratic form on packed fp32 pairs
    auto step_general = [&](const RecView rec, uint32_t zb, bool active) {
        if (!active) return;
        const float4 g0 = rec.chunk(0), g1 = rec.chunk(1), g2c = rec.chunk(2);
        const float2 g2 = make_float2(g2c.x, g2c.y);
        float wv[VOX];
#pragma unroll
        for (int h2 = 0; h2 < VOX / 2; ++h2) {
            const int v0 = 2 * h2, v1 = v0 + 1;
            const float2 dx = fadd2(make_float2(g0.x, g0.x), make_float2(-px[v0], -px[v1]));
            const float2 dy = fadd2(make_float2(g0.y, g0.y), make_float2(-py[v0], -py[v1]));
            const float2 dz = fadd2(make_float2(g0.z, g0.z), make_float2(-pz[v0], -pz[v1]));
            float2 t1 = fmul2(make_float2(g1.x, g1.x), dx);
            t1 = ffma2(make_float2(g1.w, g1.w), dy, t1);
            t1 = ffma2(make_float2(g2.y, g2.y), dz, t1);
            float2 t2 = fmul2(make_float2(g1.y, g1.y), dy);
            t2 = ffma2(make_float2(g2.x, g2.x), dz, t2);
            float2 q = fmul2(t1, dx);
            q = ffma2(t2, dy, q);
            q = ffma2(fmul2(make_float2(g1.z, g1.z), dz), dz, q);
            const float E0 = ((zb >> v0) & 1u) ? ex2_approx(q.x) : 0.f;
            const float E1 = ((zb >> v1) & 1u) ? ex2_approx(q.y) : 0.f;
            wv[v0] = PROB ? g0.w * E0 : E0;
            wv[v1] = PROB ? g0.w * E1 : E1;
            if (PROB) {
                zsum[v0] += wv[v0]; dens[v0] += E0; keep[v0] *= (1.f - E0);
                zsum[v1] += wv[v1]; dens[v1] += E1; keep[v1] *= (1.f - E1);
            }
        }
        accumulate(rec, g2c, wv);
    };
    // the column form is chosen per CTA (one vote); a CTA with any other thread takes the general form for all
    const bool all_column = __syncthreads_and((column && (PROB || D <= 32)) ? 1 : 0) != 0;
    walk_tile<C>(pin, sm, binX0, binY0, binZ0, my_zshift, all_column, step_column, step_general);
#ifdef GF_RENDER_TIMING
    const long long t_epi = clock64();
#endif

    // ---- epilogue ----------------------------------------------------------------------------------
    const RenderParams p = with_sample_outputs(pin, pb, sample);
    float out[VOX][C];
#pragma unroll
    for (int v = 0; v < VOX; ++v)
#pragma unroll
        for (int c = 0; c < C; ++c) out[v][c] = (c & 1) ? acc[v][c >> 1].y : acc[v][c >> 1].x;
    if (PROB) {
#pragma unroll
        for (int v = 0; v < VOX; ++v) {
            if (zsum[v] > 1e-9f) {
#pragma unroll
                for (int c = 0; c < C; ++c) out[v][c] = __fdiv_rn(out[v][c], zsum[v]);
            } else {
#pragma unroll
                for (int c = 0; c < C; ++c) out[v][c] = (c < C - 1) ? static_cast<float>(1.0 / (C - 1)) : 0.f;
            }
        }
    }
    if (p.out.argmax && live) {   // fused occupancy prediction (lowest index on ties)
        uint32_t packed = 0;
#pragma unroll
        for (int v = 0; v < VOX; ++v) packed |= static_cast<uint32_t>(argmax_of<C>(out[v])) << (8 * v);
        if (vec_ok) {
            *reinterpret_cast<uint32_t *>(p.out.argmax + n0) = packed;
        } else {
#pragma unroll
            for (int v = 0; v < VOX; ++v)
                if (vox_ok[v]) p.out.argmax[n0 + v] = static_cast<uint8_t>(packed >> (8 * v));
        }
    }
    if (p.out.ce_partials) {
        // softmax cross-entropy of my voxels against the labels: CE_ssc_loss = nn.CrossEntropyLoss(weight, ignore_index=255,
        // reduction='mean') (loss/occupancy_loss.py:164-178): this CTA's (sum w[y] * nll, sum w[y]), combined in a fixed order.
        float s_nll = 0.f, s_w = 0.f;
        if (live) {
#pragma unroll
            for (int v = 0; v < VOX; ++v) {
                const int y = (vox_ok[v] && !((stray >> v) & 1u)) ? static_cast<int>(p.out.labels[n0 + v]) : 255;
                if (y < C) {
                    float mx = out[v][0];
#pragma unroll
                    for (int c = 1; c < C; ++c) mx = fmaxf(mx, out[v][c]);
                    float se = 0.f, xy = out[v][0];
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        se += ex2_approx((out[v][c] - mx) * kLog2e);
                        xy = (c == y) ? out[v][c] : xy;
                    }
                    const float wy = p.out.class_weights ? __ldg(p.out.class_weights + y) : 1.f;
                    s_nll = fmaf(wy, mx + __log2f(se) * 0.6931471805599453f - xy, s_nll);
                    s_w += wy;
                }
            }
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            s_nll += __shfl_xor_sync(0xffffffffu, s_nll, o);
            s_w += __shfl_xor_sync(0xffffffffu, s_w, o);
        }
        if (lane == 0) { sm.ce[warp][0] = s_nll; sm.ce[warp][1] = s_w; }
        __syncthreads();
        if (tid == 0) {
            float a = 0.f, b = 0.f;
#pragma unroll
            for (int w = 0; w < kRenderThreads / 32; ++w) { a += sm.ce[w][0]; b += sm.ce[w][1]; }
            const long long cta = (static_cast<long long>(blockIdx.z - sample * pb.nbx) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
            p.out.ce_partials[2 * cta] = a;
            p.out.ce_partials[2 * cta + 1] = b;
        }
    }
    // [N, C] logits through the shared tile and bulk copies when that writes exactly what the direct stores would:
    // 16-byte aligned rows, whole z chunks (each column of the bin is then one contiguous run of kBinZ * C floats) and
    // no stray point in the CTA (render_one_point overwrites a stray row with ordinary stores after the direct ones).
    // A thread's direct stores would touch 32 lines per warp instruction at a 4*C*4-byte stride; the copies write
    // whole lines, and the CTA exits once the tile has been read instead of after issuing every store.
    bool bulk = p.out.logits && vec_ok && D % kBinZ == 0;
    if (bulk) {
        __syncthreads();   // every warp is done with the walk buffers the tile overwrites
        uint32_t any_stray = 0;
#pragma unroll
        for (int w = 0; w < kRenderThreads / 32; ++w) any_stray |= sm.stray_warp[w];
        bulk = any_stray == 0;
    }
    if (bulk) {
        if (live) {
            float *dst = &sm.tile[lx * kBinY + ly][VOX * C * lq];
            float flat[VOX * C];
#pragma unroll
            for (int v = 0; v < VOX; ++v)
#pragma unroll
                for (int c = 0; c < C; ++c) flat[v * C + c] = out[v][c];
#pragma unroll
            for (int i = 0; i < VOX * C / 4; ++i)
                st_shared16(dst + 4 * i, make_float4(flat[4 * i], flat[4 * i + 1], flat[4 * i + 2], flat[4 * i + 3]));
        }
        fence_proxy_async_shared();
        __syncthreads();
        if (warp == 0) {   // lane l copies column l of the bin
            const int cx = binX0 + lane / kBinY, cy = binY0 + lane % kBinY;
            if (cx < H && cy < W)
                bulk_copy_s2g(p.out.logits + ((static_cast<long long>(cx) * W + cy) * D + binZ0) * C, &sm.tile[lane][0],
                              kBinZ * C * sizeof(float));
            bulk_commit_wait_read();
        }
    }
    if (live) {
        if (vec_ok) {
            if (p.out.logits && !bulk) {
                float *dst = p.out.logits + n0 * C;
                float flat[VOX * C];
#pragma unroll
                for (int v = 0; v < VOX; ++v)
#pragma unroll
                    for (int c = 0; c < C; ++c) flat[v * C + c] = out[v][c];
                // n0 % 4 == 0, so the 4*C floats start 16-byte aligned
#pragma unroll
                for (int i = 0; i < VOX * C / 4; ++i)
                    __stcs(reinterpret_cast<float4 *>(dst) + i,
                           make_float4(flat[4 * i], flat[4 * i + 1], flat[4 * i + 2], flat[4 * i + 3]));
            }
            if (p.out.logits_cn) {   // class-major: my 4 voxels are 16 contiguous bytes of every class row
#pragma unroll
                for (int c = 0; c < C; ++c)
                    __stcs(reinterpret_cast<float4 *>(p.out.logits_cn + static_cast<long long>(c) * p.d.N + n0),
                           make_float4(out[0][c], out[1][c], out[2][c], out[3][c]));
            }
            if (PROB) {
                __stcs(reinterpret_cast<float4 *>(p.out.bin_logits + n0), make_float4(1.f - keep[0], 1.f - keep[1], 1.f - keep[2], 1.f - keep[3]));
                __stcs(reinterpret_cast<float4 *>(p.out.density + n0), make_float4(dens[0], dens[1], dens[2], dens[3]));
                __stcs(reinterpret_cast<float4 *>(p.out.probability + n0), make_float4(zsum[0], zsum[1], zsum[2], zsum[3]));
            }
        } else {
#pragma unroll
            for (int v = 0; v < VOX; ++v)
                if (vox_ok[v]) {
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        if (p.out.logits) p.out.logits[(n0 + v) * C + c] = out[v][c];
                        if (p.out.logits_cn) p.out.logits_cn[static_cast<long long>(c) * p.d.N + n0 + v] = out[v][c];
                    }
                    if (PROB) {
                        p.out.bin_logits[n0 + v] = 1.f - keep[v];
                        p.out.density[n0 + v] = dens[v];
                        p.out.probability[n0 + v] = zsum[v];
                    }
                }
        }
        // points that are not in canonical voxel order: exact per-point evaluation overwrites their rows
        if (stray) {
#pragma unroll
            for (int v = 0; v < VOX; ++v)
                if (vox_ok[v] && ((stray >> v) & 1u)) render_one_point<C, PROB>(p, n0 + v, px[v], py[v], pz[v]);
        }
    }
#ifdef GF_RENDER_TIMING
    if (tid == 0) {
        unsigned long long *t = reinterpret_cast<unsigned long long *>(p.ws.flags + 4);   // bytes 16..47 of the status block
        atomicAdd(t + 0, sm.t_phase[0]);
        atomicAdd(t + 1, sm.t_phase[1]);
        atomicAdd(t + 2, sm.t_phase[2]);
        atomicAdd(t + 3, static_cast<unsigned long long>(clock64() - t_epi));
        for (int i = 4; i < 8; ++i) atomicAdd(t + i, sm.t_phase[i]);   // bytes 48..79 (the status block is 256 bytes)
    }
#endif
}

// ------------------------------------------------------------------------------------------------
// generic path: arbitrary points
// ------------------------------------------------------------------------------------------------
// Launched only when N != H*W*D, the case for which gf_splat_forward seeds the status word with GF_FLAG_GENERIC_PATH
// (written by list_kernel), so the flag needs no check here.
template <int C, bool PROB>
__global__ void __launch_bounds__(256) render_points_kernel(const RenderParams pb) {
    const RenderParams p = with_sample_outputs(sample_params(pb, blockIdx.y), pb, blockIdx.y);
    for (long long n = blockIdx.x * 256ll + threadIdx.x; n < p.d.N; n += 256ll * gridDim.x)
        render_one_point<C, PROB>(p, n, p.pts[3 * n], p.pts[3 * n + 1], p.pts[3 * n + 2]);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
template <int C, bool PROB>
static int launch_render_t(const RenderParams &rp, bool tile_path, int num_sms, cudaStream_t stream) {
    const int B = batch_of(rp.d);
    if (tile_path) {
        GF_REQUIRE(rp.nby <= 65535 && static_cast<long long>(rp.nbx) * B <= 65535, GF_ERR_UNSUPPORTED,
                   "splat: grid x batch too large for the render launch");
        const dim3 grid(rp.nzc, rp.nby, rp.nbx * B);
        const bool timed = g_ev_before && g_ev_after;
        if (timed) GF_CUDA_TRY(cudaEventRecord(g_ev_before, stream));
        if (timed) {   // kernel timed alone: plain stream order
            render_tile_kernel<C, PROB><<<grid, kRenderThreads, sizeof(RenderSmem<C>), stream>>>(rp);
        } else {
            GF_CUDA_TRY(launch_chained(render_tile_kernel<C, PROB>, grid, dim3(kRenderThreads), sizeof(RenderSmem<C>), stream, rp));
        }
        GF_CUDA_TRY(cudaGetLastError());
        if (timed) GF_CUDA_TRY(cudaEventRecord(g_ev_after, stream));
        return GF_OK;   // stray points were handled inside the tile kernel
    }
    const long long want = (static_cast<long long>(rp.d.N) + 255) / 256;
    const int gx = static_cast<int>(want < 8ll * num_sms ? (want > 0 ? want : 1) : 8ll * num_sms);
    render_points_kernel<C, PROB><<<dim3(gx, B), 256, 0, stream>>>(rp);
    GF_CUDA_TRY(cudaGetLastError());
    return GF_OK;
}

// render CTAs of the tile path per sample (= rows of out.ce_partials per sample)
int render_ctas_per_sample(const gf_splat_desc &d) {
    return ((d.D + kBinZ - 1) / kBinZ) * ((d.W + kBinY - 1) / kBinY) * ((d.H + kBinX - 1) / kBinX);
}

int launch_render(const gf_splat_desc &d, const gf_splat_inputs &in, const gf_splat_outputs &out,
                  const SplatWorkspace &ws, bool tile_path, int num_sms, cudaStream_t stream) {
    RenderParams rp;
    rp.d = d;
    rp.pts = in.pts;
    rp.points_int = in.points_int;
    rp.out = out;
    rp.ws = ws;
    rp.nby = (d.W + kBinY - 1) / kBinY;
    rp.nzc = (d.D + kBinZ - 1) / kBinZ;
    rp.nbx = (d.H + kBinX - 1) / kBinX;
    rp.ce_rows = render_ctas_per_sample(d);
    // 16-byte vector accesses need D % 4 == 0 (a thread's z quad is then 4 consecutive points of every tensor) and
    // 16-byte aligned tensors; anything else takes the scalar loads / stores of the same kernel
    auto al16 = [](const void *q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
    rp.vec_ok = (d.D & 3) == 0 && al16(in.pts) && al16(out.logits) && al16(out.logits_cn) && al16(out.bin_logits) &&
                al16(out.density) && al16(out.probability) && (reinterpret_cast<uintptr_t>(out.argmax) & 3u) == 0;
    const bool prob = d.variant == GF_SPLAT_PROB;
    return dispatch_classes(d.C, "splat", [&](auto cc) {
        constexpr int C = decltype(cc)::value;
        return prob ? launch_render_t<C, true>(rp, tile_path, num_sms, stream)
                    : launch_render_t<C, false>(rp, tile_path, num_sms, stream);
    });
}

}  // namespace gf
