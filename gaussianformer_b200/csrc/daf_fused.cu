// Deformable aggregation fused with its caller's pre- and post-processing (SURVEY.md 8f-2b):
//
//   weights[~mask] = -inf; weights[all_miss] = 0; weights = softmax over (key point, camera, level)
//   weights *= 1 - all_miss; features = DAF(feat, points_2d, weights); features = features.sum(key points)
//
// i.e. model/encoder/gaussian_encoder/deformable_module.py:213-228 and :242 around the op call at :226.
// The reference materialises the normalised weights ([B, A*K, M, L, Gr], 88 MB at the nuScenes shape),
// reads them back in the op, writes one feature vector per KEY POINT ([B, A*K, C], 118 MB) and reduces
// that over the K key points in another kernel.  Here one warp owns one ANCHOR:
//
//   pass 1/2  the warp reads the anchor's K*M*L*Gr raw logits once, coalesced (lane -> group lane % Gr),
//             and keeps max and 1/sum per group: the normalised weight of an entry is then
//             exp2(logit*log2e - max*log2e) / sum, evaluated where it is used and never stored;
//   sampling  the K key points are visited in turn with the pair setup and visit of daf_fast_kernel
//             (setup_pairs / visit_pairs, daf_pair.cuh); the accumulator stays in registers across key
//             points and is written once per anchor ([B, A, C]: K times fewer output bytes).
//
// Backward uses  sum_e w_e * dL/dw_e = sum_{c in group} dL/dout_c * out_c  (out = sum_e w_e * val_e), so
// the softmax gradient  w_e * (dL/dw_e - that sum)  needs no second pass over the samples: every entry first
// receives -w_e * S (the value for an entry whose sample is zero) in one coalesced sweep and the visited
// (camera, level) pairs overwrite theirs.
#include "daf_pair.cuh"

namespace gf {

template <bool BACKWARD, class T, bool FEAT_GRAD = true>
__global__ void __launch_bounds__(kDafThreads, BACKWARD ? 3 : 4) daf_fused_kernel(const DafFusedParams p) {
    constexpr int kWarps = kDafThreads / 32;
    __shared__ int lh[kMaxLevels], lw[kMaxLevels], ls[kMaxLevels];
    __shared__ __align__(16) PairSetup s_pair[kWarps][32];
    __shared__ float s_mlog[kWarps][32], s_inv[kWarps][32], s_dot[kWarps][32];
    load_level_table(p.d, p.shape, p.start, lh, lw, ls);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int C = p.d.num_embeds, M = p.d.num_cams, L = p.d.num_scale, Gr = p.d.num_groups, F = p.d.num_feat;
    const int K = p.K, npair = M * L, LG = L * Gr;
    const int nE = K * npair * Gr;                       // logits of one anchor
    const int gdim = C / Gr, lanes_per_group = gdim / 4;
    const int A = p.d.num_pts / K;
    const long long nanchor = static_cast<long long>(p.d.batch) * A;
    const long long warps = static_cast<long long>(gridDim.x) * kWarps;
    PairSetup *mine = s_pair[warp];
    const int my_cam = lane / L, my_lv = lane - my_cam * L;
    const int eg = lane & (Gr - 1);                      // group of the entries this lane sweeps (Gr | 32)
    // point-mask index of entry e = lane + 32*it is e / (L*Gr); when L*Gr divides 32 that is it*pm_step + pm_sub
    // without a division in the sweeps (L*Gr = 16 at the shipped shapes)
    const bool pm_fast = LG <= 32 && (32 % LG) == 0;
    const int pm_step = pm_fast ? 32 / LG : 0, pm_sub = pm_fast ? lane / LG : 0;

    for (long long ba = static_cast<long long>(blockIdx.x) * kWarps + warp; ba < nanchor; ba += warps) {
        const int b = static_cast<int>(ba / A);
        const float *wl = p.logits + ba * nE;
        const uint8_t *pm = p.pmask ? p.pmask + ba * K * M : nullptr;
        const uint8_t *wm = p.wmask ? p.wmask + ba * nE : nullptr;

        // ---- softmax statistics of the anchor: max and 1/sum per group over its K*M*L unmasked entries -----
        if (!BACKWARD) {
            float mx = -INFINITY;
            for (int e = lane, it = 0; e < nE; e += 32, ++it) {
                const bool on = (!pm || pm[pm_fast ? it * pm_step + pm_sub : e / LG]) && (!wm || wm[e]);
                if (on) mx = fmaxf(mx, __ldg(wl + e));
            }
            for (int o = Gr; o < 32; o <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            const float mlog = (mx == -INFINITY) ? 0.f : mx * kLog2e;
            float sum = 0.f;
            for (int e = lane, it = 0; e < nE; e += 32, ++it) {
                const bool on = (!pm || pm[pm_fast ? it * pm_step + pm_sub : e / LG]) && (!wm || wm[e]);
                if (on) sum += softmax_term(__ldg(wl + e), mlog);
            }
            for (int o = Gr; o < 32; o <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            // a group with every entry masked ("all_miss", deformable_module.py:215-218,228) gets weight 0 everywhere
            const float inv = sum > 0.f ? __fdividef(1.f, sum) : 0.f;
            if (lane < Gr) {
                s_mlog[warp][lane] = mlog;
                s_inv[warp][lane] = inv;
                *reinterpret_cast<float2 *>(p.stats + (ba * Gr + lane) * 2) = make_float2(mlog, inv);
            }
        } else {
            if (lane < Gr) {
                const float2 st = __ldg(reinterpret_cast<const float2 *>(p.stats + (ba * Gr + lane) * 2));
                s_mlog[warp][lane] = st.x;
                s_inv[warp][lane] = st.y;
            }
            // S_g = sum_{c in g} dL/dout_c * out_c  ( = sum_e w_e * dL/dw_e )
            for (int c0 = lane * 4; c0 < C; c0 += 128) {
                const float4 g = __ldg(reinterpret_cast<const float4 *>(p.grad_out + ba * C + c0));
                const float4 o4 = __ldg(reinterpret_cast<const float4 *>(p.out_saved + ba * C + c0));
                float s = g.x * o4.x + g.y * o4.y + g.z * o4.z + g.w * o4.w;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1)
                    if (o < lanes_per_group) s += __shfl_xor_sync(0xffffffffu, s, o);
                if ((lane & (lanes_per_group - 1)) == 0) s_dot[warp][c0 / gdim] = s;
            }
        }
        __syncwarp();
        if (BACKWARD) {
            // every entry as if its sample were zero: dL/dlogit_e = -w_e * S_g; visited pairs overwrite theirs below
            const float mlog = s_mlog[warp][eg], inv = s_inv[warp][eg], S = s_dot[warp][eg];
            for (int e = lane, it = 0; e < nE; e += 32, ++it) {
                const bool on = (!pm || pm[pm_fast ? it * pm_step + pm_sub : e / LG]) && (!wm || wm[e]);
                const float w = on ? softmax_weight(__ldg(wl + e), mlog, inv, nullptr, e) : 0.f;   // on holds both masks
                p.grad_logits[ba * nE + e] = -w * S;
            }
            __syncwarp();
        }

        // ---- sampling: K key points accumulate into one register vector per lane -----------------------------
        const T *featb = static_cast<const T *>(p.feat) + static_cast<long long>(b) * M * F * C;
        float *gfeatb = p.grad_feat + static_cast<long long>(b) * M * F * C;
        for (int c0 = lane * 4; c0 < C; c0 += 128) {
            const int grp = c0 / gdim;
            const float mlog = s_mlog[warp][grp], inv = s_inv[warp][grp];
            const float S = BACKWARD ? s_dot[warp][grp] : 0.f;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            float4 gout = make_float4(0.f, 0.f, 0.f, 0.f);
            if (BACKWARD) gout = __ldg(reinterpret_cast<const float4 *>(p.grad_out + ba * C + c0));
            for (int k = 0; k < K; ++k) {
                const long long bp = ba * K + k;
                const uint32_t visible = setup_pairs(p.d, p.loc, lh, lw, ls, bp, lane, my_cam, my_lv, pm ? pm + k * M : nullptr, mine);
                const float *wpt = wl + k * npair * Gr;
                const uint8_t *wmk = wm ? wm + k * npair * Gr : nullptr;
                visit_pairs<BACKWARD, FEAT_GRAD>(
                    mine, visible, featb, gfeatb, c0, lane, lanes_per_group, gout, p.grad_loc, bp, M, acc,
                    [=](int pr) { const int widx = pr * Gr + grp; return softmax_weight(__ldg(wpt + widx), mlog, inv, wmk, widx); },
                    // dL/dw_e = sampled value . g, then through the softmax
                    [glg = p.grad_logits, ba, nE, k, npair, Gr, grp, S](int pr, float wt, float gw) {
                        glg[ba * nE + static_cast<long long>(k) * npair * Gr + pr * Gr + grp] = wt * (gw - S);
                    });
                __syncwarp();   // the next key point overwrites this warp's setup slots
            }
            if (!BACKWARD) *reinterpret_cast<float4 *>(p.out + ba * C + c0) = acc;
        }
        __syncwarp();           // ... and the next anchor its statistics
    }
}

bool daf_fused_supported(const gf_daf_desc &d, int K) {
    if (!daf_vec4_ok(d)) return false;
    const int Gr = d.num_groups;
    if (Gr > 32 || (Gr & (Gr - 1)) != 0) return false;
    if (K < 1 || d.num_pts % K != 0) return false;
    return static_cast<long long>(K) * d.num_cams * d.num_scale * Gr < (1ll << 31);
}

int launch_daf_fused(const DafFusedParams &p, int dtype, DafPass pass, int num_sms, cudaStream_t stream) {
    const long long nanchor = static_cast<long long>(p.d.batch) * (p.d.num_pts / p.K);
    if (nanchor == 0) return GF_OK;
    const int grid = daf_grid(nanchor, num_sms);
    return dispatch_feat_dtype(dtype, "daf fused", [&](auto tag) {
        using T = typename decltype(tag)::type;
        if (pass == DafPass::kForward) daf_fused_kernel<false, T><<<grid, kDafThreads, 0, stream>>>(p);
        else if (pass == DafPass::kBackward) daf_fused_kernel<true, T><<<grid, kDafThreads, 0, stream>>>(p);
        else daf_fused_kernel<true, T, false><<<grid, kDafThreads, 0, stream>>>(p);
        GF_CUDA_TRY(cudaGetLastError());
        return GF_OK;
    });
}

}  // namespace gf
