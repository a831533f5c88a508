/*
 * glom_b200_track.h -- island tracks through time over the islands of glom_b200_islands (libglom_b200.so).
 *
 * GLOM's claim is that islands persist: through the iterations of one image as they form, and across consecutive frames
 * of a slow video.  glom_b200_islands labels each slab on its own; this call links each level's islands at slab t - 1
 * to those at slab t and gives every island a track id.  The conventions of glom_b200.h hold: device pointers owned by
 * the caller, no allocation, no synchronisation, 0 or a negative glom_b200_status with the text in
 * glom_b200_last_error().
 */
#ifndef GLOM_B200_TRACK_H_
#define GLOM_B200_TRACK_H_

#include "glom_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Tracks of outer * inner label sequences of `times` slabs each.
 *
 * labels (outer, times, inner, levels, n) int32: island labels as glom_b200_islands writes them for states (outer,
 *   times, inner, n, levels, dim), so time may be any leading dimension of the states with no copy.  A sequence is one
 *   (outer, inner) index, and "slab t" its index t along `times`.  Membership is that of glom_b200_tree.h: patch i is a
 *   member of island j = lab[l, i] when 0 <= j <= i and lab[l, j] == j; a patch that is no member (garbage labels:
 *   negative, >= n, or pointing at a non-root) is skipped by every output below.  A root is a patch with members.
 *
 * Outputs, each (outer, times, inner, levels, n) int32, per sequence and level (overlap(j, k) = |{i member of j at
 * slab t and of k at slab t - 1}|):
 *   prev     at a root j of slab t >= 1: the label k at slab t - 1 with the largest overlap(j, k), ties to the smallest
 *            k; -1 at non-roots, at t = 0 and where no member of j is a member of anything at t - 1
 *   overlap  overlap(j, prev) where prev >= 0, else 0
 *   next     at a root k of slab t <= times - 2: the label j at slab t + 1 with the largest overlap, ties to the
 *            smallest j; -1 elsewhere and at t = times - 1
 *   track    per patch, the track id of its island; -1 for a non-member.  Island j at slab t continues the track of
 *            k = prev[t][j] when the two are each other's best match (next[t-1][k] == j); otherwise it starts the new
 *            track t * n + j.  An id decodes to its birth: slab id / n, root id % n.  At t = 0, track is the label.
 *            In a split the part with the larger overlap keeps the track; in a merge the island with the larger
 *            overlap carries its track on and the other track ends.
 *
 * Limits are those of glom_b200_island_tree: 1 <= outer * times * inner <= 65535 slabs, 1 <= n <= 8192,
 * 1 <= levels <= 65535, so a track id is below 65535 * 8192 < 2^31.  labels and the outputs must be 4-byte aligned.
 * Every output is written in full.
 *
 * Determinism: every result is a pure function of the labels, bit-identical from run to run and for every SM-count
 * target.  Overlaps are integer counts (order-free); prev and next are maxima of packed (overlap, ~label) keys.
 *
 * Work: two CUDA-core kernels that read labels only.  The pair kernel runs one block per (slab, level) and counts the
 * (island at t, island at t - 1) pairs in a shared-memory hash table; the track kernel runs one block per (sequence,
 * level) and walks t in order.  Argument errors are returned before any device query. */
GLOM_B200_API int glom_b200_island_track(const int32_t* labels, int outer, int times, int inner, int n, int levels,
                                         int32_t* prev, int32_t* overlap, int32_t* next, int32_t* track, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* GLOM_B200_TRACK_H_ */
