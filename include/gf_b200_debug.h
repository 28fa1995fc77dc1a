/*
 * gf_b200_debug.h -- measurement hooks of libgf_b200.so.  NOT part of the drop-in boundary (include/gf_b200.h): nothing
 * here replaces a reference interface, and a product caller never needs it.  bench.py uses it for the roofline line.
 */
#ifndef GF_B200_DEBUG_H_
#define GF_B200_DEBUG_H_

#include "gf_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* When both events are non-NULL (cudaEvent_t created with timing enabled), every following gf_splat_forward of the
 * CALLING THREAD records them on its stream immediately before / after the render kernel and launches that kernel in
 * plain stream order (no programmatic overlap with its predecessors), so that it can be timed alone inside a normal
 * run.  Thread-local state; pass NULLs to switch it off. */
int gf_debug_set_render_events(void *before, void *after);

/* Random row gather over a table (row i = row_floats floats, a multiple of 128; idx[n] int32 row numbers, device):
 * the access pattern of the sampling op without its arithmetic.  With an L2-resident table the achieved
 * n * row_floats * 4 bytes / time is the L2 -> SM gather bandwidth that bounds gf_daf_forward on uncorrelated
 * sampling points (tools/daf_experiments.py). */
int gf_debug_gather_probe(const float *table, const int32_t *idx, int64_t n, int32_t row_floats, float *sink,
                          gf_stream_t stream);

/* Launch plan of every following splat backward in the process: slot_budget >= 0 replaces the per-sample slot budget
 * of the deterministic bin route (and with it gf_splat_backward_workspace_bytes_ex), num_sms > 0 the SM count the
 * launch grids are sized for.  Negative / 0: back to the defaults.  For tests of the slot-overflow hand-over and of
 * results that must not depend on the GPU size. */
int gf_debug_splat_backward_plan(int64_t slot_budget, int32_t num_sms);

/* Which route produced the gradients of the last GF_BWD_DETERMINISTIC gf_splat_backward_ex that used `workspace`:
 * host_route[b] (b < batch) receives one of the values below.  Synchronises the stream. */
#define GF_DEBUG_ROUTE_BIN 0u            /* bin-centric kernel, slot rows */
#define GF_DEBUG_ROUTE_SLOT_OVERFLOW 1u  /* canonical points, but the slots did not fit: Gaussian-centric chain */
#define GF_DEBUG_ROUTE_STRAY_POINTS 2u   /* the bin kernel found a point out of canonical order: Gaussian-centric chain */
#define GF_DEBUG_ROUTE_GAUSSIAN 3u       /* the bin kernel does not apply to the call: Gaussian-centric chain */
int gf_debug_splat_backward_route(const gf_splat_desc *desc, const void *workspace, gf_stream_t stream,
                                  uint32_t *host_route);

/* The SM count every following deformable-aggregation call in the process sizes its launch grids for (forwards and
 * backwards, both routes); <= 0: back to the device's.  For tests of results that must not depend on the GPU size. */
int gf_debug_daf_plan(int32_t num_sms);

/* The sorted order of the last gf_occ_loss that used `workspace` (same desc): *host_num_v = |V|, host_present[c]
 * (C bytes) whether class c was present, and for each present class row c of host_order [C, B * N] receives, in its
 * first |V| entries, the positions in V of the errors in sorted order (other entries are left as they are).
 * Synchronises the stream. */
int gf_debug_occ_loss_order(const gf_occ_loss_desc *desc, const void *workspace, gf_stream_t stream,
                            int32_t *host_order, int32_t *host_num_v, uint8_t *host_present);

/* The rulebook gf_subm_conv_rulebook left in `workspace` (same desc): *host_num_voxels = M, the occupied voxels;
 * host_slot[N] the voxel slot of every row (slots number the occupied voxels in ascending (b, x, y, z) order; -1 for an
 * invalid row); host_rep[N] the representative row of every slot in its first M entries; host_nbr [N, k^3] in its
 * first M rows the slot of the neighbour at every offset, or -1.  Entries past M are left as they are.  Synchronises
 * the stream. */
int gf_debug_subm_conv_neighbors(const gf_subm_conv_desc *desc, const void *workspace, gf_stream_t stream,
                                 int32_t *host_num_voxels, int32_t *host_slot, int32_t *host_rep, int32_t *host_nbr);

#ifdef __cplusplus
}
#endif
#endif /* GF_B200_DEBUG_H_ */
