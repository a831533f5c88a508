// Island tracks through time over the island labels (include/glom_b200_track.h).
//
// Input: label maps (outer, times, inner, L, n) int32 as glom_b200_islands writes them for states (outer, times, inner,
// n, L, d).  A sequence is one (outer, inner) index; slab t is its index t along `times`.  Per (sequence, level):
//   prev[t][j]    at a root j of slab t >= 1, the label k at t - 1 with the largest overlap |{i member of j at t and of
//                 k at t - 1}|, ties to the smallest k; -1 elsewhere
//   overlap[t][j] that overlap where prev >= 0, else 0
//   next[t][k]    at a root k of slab t <= times - 2, the label j at t + 1 with the largest overlap, ties to the smallest
//                 j; -1 elsewhere
//   track[t][i]   the track id of patch i's island, -1 for a non-member.  Island j at t continues the track of
//                 k = prev[t][j] when the two are each other's best match (next[t-1][k] == j); otherwise it starts the
//                 track t * n + j, which decodes to its birth slab and root.
//
// Membership and the pair table are those of the part-whole trees (island_pairs.cuh): garbage labels are skipped and
// never index outside [0, n).
//
// Determinism: the overlaps are integer counts (order-free shared-memory atomics) and prev / next are maxima of packed
// (overlap, ~label) keys, so the largest overlap wins and ties go to the smallest label in any atomic order.  The track
// walk is a fixed sequence of block-wide phases.  The grids are (L, slabs) and (L, sequences) and depend on nothing
// else, so no result depends on the SM count.
#include "engine.h"
#include "island_pairs.cuh"

namespace glom {

namespace {

constexpr int kTrackThreads = 256;

}  // namespace

// One block per (level l, slab s), t = s's index along `times`: for t >= 1 the pair table of (island at t, island at
// t - 1) gives prev / overlap of slab t and next of slab t - 1; slab 0 gets the prev / overlap defaults and slab
// times - 1 the next default.  So every element of the three outputs is written by exactly one block.
// Shared memory: table[slots] of (pair key + 1) << 32 | overlap with pair key = j * n + k < 2^26, best_k[n] (per j at
// t, packed), best_j[n] (per k at t - 1, packed).
__global__ void __launch_bounds__(kTrackThreads)
island_pair_kernel(const int* __restrict__ labels, int times, int inner, int n, int slots, int* __restrict__ prev,
                   int* __restrict__ overlap, int* __restrict__ next) {
  extern __shared__ unsigned long long pair_sm[];
  unsigned long long* table = pair_sm;                                   // [slots]
  unsigned* best_k = reinterpret_cast<unsigned*>(table + slots);         // [n]
  unsigned* best_j = best_k + n;                                         // [n]
  const int l = blockIdx.x, L = gridDim.x;
  const int t = (int)((blockIdx.y / (unsigned)inner) % (unsigned)times);
  const size_t o = ((size_t)blockIdx.y * L + l) * n;                     // slab t, level l
  const size_t o_prev = o - (size_t)inner * L * n;                       // slab t - 1, level l (valid only when t >= 1)
  if (t == times - 1)
    for (int k = threadIdx.x; k < n; k += blockDim.x) next[o + k] = -1;
  if (t == 0) {
    for (int j = threadIdx.x; j < n; j += blockDim.x) { prev[o + j] = -1; overlap[o + j] = 0; }
    return;
  }
  const int* lab = labels + o;
  const int* old = labels + o_prev;
  for (int s = threadIdx.x; s < slots; s += blockDim.x) table[s] = 0ull;
  for (int j = threadIdx.x; j < n; j += blockDim.x) { best_k[j] = 0u; best_j[j] = 0u; }
  __syncthreads();
  const unsigned mask = (unsigned)slots - 1;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int j = member_of(lab, i);
    if (j < 0) continue;
    const int k = member_of(old, i);
    if (k < 0) continue;
    pair_insert(table, mask, (unsigned)j * (unsigned)n + (unsigned)k);
  }
  __syncthreads();
  pair_sweep(table, slots, n, [&](unsigned j, unsigned k, unsigned ov) {
    atomicMax(&best_k[j], pack_best(ov, k));
    atomicMax(&best_j[k], pack_best(ov, j));
  });
  __syncthreads();
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const unsigned b = best_k[j];
    prev[o + j] = best_label(b);
    overlap[o + j] = best_overlap(b);
    next[o_prev + j] = best_label(best_j[j]);
  }
}

// One block per (level l, sequence q), walking t = 0 .. times - 1 in order.  A root's id at t is stored at its own
// patch: (a) each root j reads k = prev[t][j] and, when next[t-1][k] == j, continues track[t-1][k], else starts
// t * n + j; (b) barrier; (c) every other patch copies its root's id, or -1 when it is no member; (d) barrier.  The
// block's own global writes of t - 1 are visible to it after the barriers.
__global__ void __launch_bounds__(kTrackThreads)
island_track_kernel(const int* __restrict__ labels, int times, int inner, int n, const int* __restrict__ prev,
                    const int* __restrict__ next, int* track) {
  const int l = blockIdx.x, L = gridDim.x;
  const int q = blockIdx.y;
  const size_t slab0 = (size_t)(q / inner) * times * inner + (size_t)(q % inner);
  const size_t stride = (size_t)inner * L * n;                           // one step along `times`
  const size_t o0 = (slab0 * L + l) * n;
  for (int t = 0; t < times; ++t) {
    const size_t o = o0 + (size_t)t * stride;
    const int* lab = labels + o;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
      if (member_of(lab, j) != j) continue;
      int id = t * n + j;
      if (t > 0) {
        const int k = prev[o + j];
        if (k >= 0 && next[o - stride + k] == j) id = track[o - stride + k];
      }
      track[o + j] = id;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int j = member_of(lab, i);
      if (j != i) track[o + i] = j < 0 ? -1 : track[o + j];
    }
    __syncthreads();
  }
}

int launch_island_track(const int* labels, int outer, int times, int inner, int n, int L, int* prev, int* overlap,
                        int* next, int* track, Launch& ln) {
  // the pair kernel's shared memory is the tree kernel's (8 * slots + 8n = 192 KB at n = 8192): opt in above 46 KB
  const int slots = tree_slots(n);
  const size_t smem = (size_t)slots * 8 + (size_t)n * 8;
  static SmemOptIn pair_optin;
  if (smem > 46 * 1024) GLOM_TRY(ln.check(pair_optin.ensure(island_pair_kernel, smem)));
  island_pair_kernel<<<dim3(L, outer * times * inner), kTrackThreads, smem, ln.st>>>(labels, times, inner, n, slots, prev,
                                                                                    overlap, next);
  GLOM_TRY(ln.launched());
  island_track_kernel<<<dim3(L, outer * inner), kTrackThreads, 0, ln.st>>>(labels, times, inner, n, prev, next, track);
  return ln.launched();
}

}  // namespace glom
