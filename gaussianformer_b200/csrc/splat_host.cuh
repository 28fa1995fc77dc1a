// Host functions of the splat pipeline that one translation unit defines and another calls, declared once here.
#pragma once
#include "common.cuh"

namespace gf {

struct BwdParams;

// Hands out consecutive 256-byte aligned regions of a workspace.  With base == nullptr only `bytes` advances, which
// sizes the workspace.
struct WorkspaceCarver {
    char *base;
    size_t bytes = 0;   // carved so far
    static size_t align(size_t n) { return (n + 255) / 256 * 256; }
    template <class T>
    T *take(size_t n) {
        T *p = base ? reinterpret_cast<T *>(base + bytes) : nullptr;
        bytes += align(n);
        return p;
    }
};

// splat_prep.cu
SplatWorkspace plan_forward_workspace(const gf_splat_desc &d, WorkspaceCarver &carve);
int launch_prep(const gf_splat_desc &d, const gf_splat_inputs &in, const SplatWorkspace &ws, uint32_t initial_flags,
                cudaStream_t stream, bool raw_records = false);

// splat_forward.cu
int launch_render(const gf_splat_desc &d, const gf_splat_inputs &in, const gf_splat_outputs &out,
                  const SplatWorkspace &ws, bool tile_path, int num_sms, cudaStream_t stream);
int render_ctas_per_sample(const gf_splat_desc &d);

// splat_backward.cu
size_t backward_workspace_bytes(const gf_splat_desc &d, uint32_t flags);
int launch_backward(const gf_splat_desc &d, const gf_splat_inputs &in, const gf_splat_grads &gr, void *workspace,
                    uint32_t flags, int num_sms, cudaStream_t stream);
// sample 0's route word (GF_DEBUG_ROUTE_*) in `workspace`; sample b's lies b * *stride bytes further
uint32_t *backward_route_words(const gf_splat_desc &d, void *workspace, size_t *stride);

// splat_backward_bin.cu
bool backward_bin_eligible(const gf_splat_desc &d, const gf_splat_inputs &in, const gf_splat_grads &gr);
// det: the deterministic slot route (bp.slots) instead of the atomic accumulation into bp.sums
int launch_backward_bin(const BwdParams &bp, bool det, cudaStream_t stream);

// cabi.cu: events recorded around the render kernel when both are set (gf_debug_set_render_events)
extern thread_local cudaEvent_t g_ev_before, g_ev_after;
// cabi.cu: the slot budget and SM count forced by gf_debug_splat_backward_plan (< 0: not forced)
long long slot_budget_override();
int num_sms_override();

}  // namespace gf
