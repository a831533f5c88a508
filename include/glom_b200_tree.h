/*
 * glom_b200_tree.h -- part-whole parse trees over the islands of glom_b200_islands (libglom_b200.so).
 *
 * GLOM's claim is that columns agree into islands at each level and that the islands of level l nest inside those of
 * level l + 1.  glom_b200_islands finds each level's islands; this call relates every level to the one above and
 * summarises each island.  The conventions of glom_b200.h hold: device pointers owned by the caller, no allocation,
 * no synchronisation, 0 or a negative glom_b200_status with the text in glom_b200_last_error().
 */
#ifndef GLOM_B200_TREE_H_
#define GLOM_B200_TREE_H_

#include "glom_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Part-whole tree of `slabs` label maps.
 *
 * labels (slabs, levels, n) int32: island labels as glom_b200_islands writes them (lab[l, i] = the smallest patch index
 *   of patch i's island at level l; a root j has lab[l, j] == j).  Patch i is a member of island j = lab[l, i] when
 *   0 <= j <= i and lab[l, j] == j, which every label map of glom_b200_islands satisfies for every patch.  A patch that
 *   is no member (garbage labels: negative, >= n, or pointing at a non-root) is skipped by every output below.
 * states (slabs, n, levels, dim) fp32, 16-byte aligned, or NULL: the states the labels were computed from.  NULL skips
 *   the three embedding outputs, which must then be NULL too; with states, all three are required.
 *
 * Outputs, per slab and level l (j ranges over patch indices; "root" = a patch with members, i.e. size > 0):
 *   size        (slabs, levels, n) int32  at a root j its member count, 0 elsewhere (each row sums to n)
 *   parent      (slabs, levels, n) int32  at a root j of level l < levels-1: the level-(l+1) label k with the largest
 *                                         overlap |{i member of j at l and of k at l+1}|, ties to the smallest k;
 *                                         -1 at non-roots, at level levels-1 and where no member has a level-(l+1) island
 *   containment (slabs, levels, n) fp32   (float)overlap / (float)size where parent >= 0, else 0
 *   nested      (slabs, levels-1) fp32    (float)(members of level-l islands with overlap == size) / (float)n; may be
 *                                         NULL when levels == 1
 *   embedding   (slabs, levels, n, dim) fp32, 16-byte aligned   at a root j: the fp32 sum of its members' level-l vectors
 *                                         in increasing patch order, divided by (float)size; 0 elsewhere
 *   member_cos  (slabs, levels, n) fp32   cosine of patch i's level-l vector with its island's embedding,
 *                                         dot / max(|x| |e|, 1e-12) as in glom_b200_islands; 0 for a non-member
 *   coherence   (slabs, levels, n) fp32   at a root: the fp32 sum of its members' member_cos in increasing patch order,
 *                                         divided by (float)size; 0 elsewhere
 *
 * Limits are those of glom_b200_islands: 1 <= slabs, levels <= 65535, 1 <= n <= 8192, dim a positive multiple of 4.
 * labels and the int32 / fp32 outputs must be 4-byte aligned.  Every output is written in full.
 *
 * Determinism: every result is a pure function of the inputs, bit-identical from run to run and for every SM-count
 * target.  Counts are integer (order-free); the parent is the maximum of the packed key (overlap, ~k); every float is
 * summed in a fixed order.
 *
 * Work: two CUDA-core kernels, one block per (slab, level) each.  The tree kernel reads labels only.  The embedding
 * kernel (only with states) reads every state vector twice (the sum, then the cosines) and writes the embedding once:
 * HBM-bound.  Argument errors are returned before any device query. */
GLOM_B200_API int glom_b200_island_tree(const int32_t* labels, const float* states, int slabs, int n, int levels, int dim,
                                        int32_t* size, int32_t* parent, float* containment, float* nested,
                                        float* embedding, float* member_cos, float* coherence, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* GLOM_B200_TREE_H_ */
