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

#ifdef __cplusplus
}
#endif
#endif /* GF_B200_DEBUG_H_ */
