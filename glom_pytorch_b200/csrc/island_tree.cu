// Part-whole parse trees over the island labels (include/glom_b200_tree.h).
//
// Input: `slabs` label maps (L levels, n patches) int32 as glom_b200_islands writes them, and optionally the state
// slabs they were computed from, (n, L, d) fp32 each.  Per (slab, level l):
//   size[j]        patches in island j (at its root j, the island's smallest patch index; 0 elsewhere)
//   parent[j]      the level-(l+1) island holding most of island j's patches, ties to the smallest label (l < L-1)
//   containment[j] overlap with the parent / size
//   nested[l]      share of patches whose level-l island lies wholly inside one level-(l+1) island
//   embedding[j]   mean of the members' level-l vectors, summed in increasing patch order
//   member_cos[i]  cosine of patch i's vector with its island's embedding; coherence[j] the members' mean of it
//
// A patch i is a member of island j = lab[i] at its level when 0 <= j <= i and lab[j] == j (the root is the smallest
// patch index, so every valid label map satisfies this for every patch).  Patches that fail are skipped everywhere:
// garbage labels never index outside [0, n) and never move a write outside the outputs.
//
// Determinism: every integer count is order-independent (shared-memory atomicAdd / atomicMax of integers); the parent
// is the maximum of the packed key (overlap << 13 | (8191 - k)), so the largest overlap wins and ties go to the
// smallest k whatever order the atomics land in.  Every float is summed in a fixed order: the embedding and coherence
// sequentially over the members in increasing patch order, the cosines' dot products in a fixed per-lane order and a
// fixed butterfly.  The grid is (L, slabs) and depends on nothing else, so no result depends on the SM count.
#include "engine.h"
#include "island_pairs.cuh"

namespace glom {

namespace {

constexpr int kTreeThreads = 256;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace

// One block per (level l, slab): sizes of level l, and for l < L-1 the overlaps with level l+1, parents, containment and
// nested.  Shared memory: cnt[n] sizes, best[n] packed parent keys, table[slots] of (pair key + 1) << 32 | overlap,
// pair key = j * n + k < 2^26.
__global__ void __launch_bounds__(kTreeThreads)
island_tree_kernel(const int* __restrict__ labels, int n, int slots, int* __restrict__ size, int* __restrict__ parent,
                   float* __restrict__ containment, float* __restrict__ nested) {
  extern __shared__ unsigned long long tree_sm[];
  unsigned long long* table = tree_sm;                                   // [slots]
  int* cnt = reinterpret_cast<int*>(table + slots);                      // [n]
  unsigned* best = reinterpret_cast<unsigned*>(cnt + n);                 // [n]
  __shared__ int contained;
  const int l = blockIdx.x, L = gridDim.x;
  const size_t o = ((size_t)blockIdx.y * L + l) * n;
  const int* lab = labels + o;
  const int* up = lab + n;                                               // level l + 1 (valid only when has_up)
  const bool has_up = l + 1 < L;
  for (int s = threadIdx.x; s < slots; s += blockDim.x) table[s] = 0ull;
  for (int j = threadIdx.x; j < n; j += blockDim.x) { cnt[j] = 0; best[j] = 0u; }
  if (threadIdx.x == 0) contained = 0;
  __syncthreads();
  const unsigned mask = (unsigned)slots - 1;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int j = member_of(lab, i);
    if (j < 0) continue;
    atomicAdd(&cnt[j], 1);
    if (!has_up) continue;
    const int k = member_of(up, i);
    if (k < 0) continue;
    pair_insert(table, mask, (unsigned)j * (unsigned)n + (unsigned)k);
  }
  __syncthreads();
  if (has_up) {
    pair_sweep(table, slots, n,
               [&](unsigned j, unsigned k, unsigned overlap) { atomicMax(&best[j], pack_best(overlap, k)); });
    __syncthreads();
  }
  int mine = 0;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const int c = cnt[j];                                                // 0 unless j is a root with members
    const unsigned b = best[j];
    const int overlap = best_overlap(b);
    size[o + j] = c;
    parent[o + j] = best_label(b);
    containment[o + j] = b ? (float)overlap / (float)c : 0.f;
    if (b && overlap == c) mine += c;
  }
  if (has_up) {
    if (mine) atomicAdd(&contained, mine);
    __syncthreads();
    if (threadIdx.x == 0) nested[(size_t)blockIdx.y * (L - 1) + l] = (float)contained / (float)n;
  }
}

// One block per (level l, slab): the members of each island in increasing patch order (a stable counting sort of the
// patches by island), then
//   phase 1: embedding[j] = (sum over members, in order) / size, one thread per (island, float4 column); zero rows at
//            non-roots
//   phase 2: member_cos[i], one warp per member (fixed-order dot products)
//   phase 3: coherence[j] = (sum of member_cos over members, in order) / size, one thread per island
// Shared memory: lab[n], cnt[n] (sizes, then the scatter cursor), off[n + 1] (exclusive scan of sizes), perm[n].
__global__ void __launch_bounds__(kTreeThreads)
island_embed_kernel(const int* __restrict__ labels, const float* __restrict__ states, int n, int d,
                    float* embedding, float* member_cos, float* __restrict__ coherence) {
  extern __shared__ int embed_sm[];
  int* lab = embed_sm;
  int* cnt = lab + n;
  int* off = cnt + n;
  int* perm = off + n + 1;
  __shared__ int warp_tot[kTreeThreads / 32];
  const int l = blockIdx.x, L = gridDim.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const size_t o = ((size_t)blockIdx.y * L + l) * n;
  for (int i = tid; i < n; i += blockDim.x) { lab[i] = labels[o + i]; cnt[i] = 0; }
  __syncthreads();
  for (int i = tid; i < n; i += blockDim.x) {
    const int j = member_of(lab, i);
    if (j >= 0) atomicAdd(&cnt[j], 1);
  }
  __syncthreads();
  // exclusive scan of cnt into off: thread t scans its contiguous chunk, the chunk totals are scanned across the block
  const int chunk = (n + blockDim.x - 1) / blockDim.x;
  const int lo = min(n, tid * chunk), hi = min(n, lo + chunk);
  int run = 0;
  for (int j = lo; j < hi; ++j) run += cnt[j];
  int incl = run;
#pragma unroll
  for (int s = 1; s < 32; s <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, s);
    if (lane >= s) incl += v;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  int base = incl - run;
  for (int w = 0; w < warp; ++w) base += warp_tot[w];
  for (int j = lo; j < hi; ++j) { off[j] = base; base += cnt[j]; }
  if (tid == blockDim.x - 1) off[n] = base;
  __syncthreads();
  for (int j = tid; j < n; j += blockDim.x) cnt[j] = 0;
  __syncthreads();
  // stable scatter by one warp, 32 patches at a time: a patch's slot is its island's cursor plus its rank among the
  // lanes of the same island
  if (warp == 0) {
    for (int b = 0; b < n; b += 32) {
      const int i = b + lane;
      const int j = i < n ? member_of(lab, i) : -1;
      const unsigned same = __match_any_sync(0xffffffffu, j);
      const int rank = __popc(same & ((1u << lane) - 1));
      if (j >= 0) perm[off[j] + cnt[j] + rank] = i;
      __syncwarp();
      if (j >= 0 && lane == 31 - __clz(same)) cnt[j] += __popc(same);
      __syncwarp();
    }
  }
  __syncthreads();
  const int d4 = d >> 2;
  const size_t pitch4 = (size_t)L * d4;                                  // float4 between consecutive patches
  const float4* x = reinterpret_cast<const float4*>(states + ((size_t)blockIdx.y * n * L + l) * d);
  float4* emb = reinterpret_cast<float4*>(embedding + o * d);
  // phase 1
  for (int j = tid / d4, c = tid % d4; j < n; c += blockDim.x, j += c / d4, c %= d4) {
    const int s = off[j], e = off[j + 1];
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (e > s) {
#pragma unroll 4
      for (int p = s; p < e; ++p) {
        const float4 v = __ldg(x + (size_t)perm[p] * pitch4 + c);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
      const float m = (float)(e - s);
      acc.x /= m; acc.y /= m; acc.z /= m; acc.w /= m;
    }
    emb[(size_t)j * d4 + c] = acc;
  }
  __syncthreads();                                       // the block's embedding rows are visible to all its threads
  // phase 2
  for (int i = warp; i < n; i += nwarps) {
    const int j = member_of(lab, i);
    float dot = 0.f, xx = 0.f, ee = 0.f;
    if (j >= 0) {
      const float4* xi = x + (size_t)i * pitch4;
      const float4* ej = emb + (size_t)j * d4;
#pragma unroll 2
      for (int c = lane; c < d4; c += 32) {
        const float4 a = __ldg(xi + c), b = ej[c];
        dot += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
        xx += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
        ee += b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w;
      }
      dot = warp_sum(dot); xx = warp_sum(xx); ee = warp_sum(ee);
    }
    if (lane == 0) member_cos[o + i] = j >= 0 ? dot / fmaxf(sqrtf(xx) * sqrtf(ee), 1e-12f) : 0.f;
  }
  __syncthreads();
  // phase 3
  for (int j = tid; j < n; j += blockDim.x) {
    const int s = off[j], e = off[j + 1];
    float acc = 0.f;
    for (int p = s; p < e; ++p) acc += member_cos[o + perm[p]];
    coherence[o + j] = e > s ? acc / (float)(e - s) : 0.f;
  }
}

int launch_island_tree(const int* labels, const float* states, int slabs, int n, int L, int d, int* size, int* parent,
                       float* containment, float* nested, float* embedding, float* member_cos, float* coherence,
                       Launch& ln) {
  // both kernels' dynamic shared memory grows with n and passes the default 48 KB per block well below the API bound
  // n = 8192 (tree: 8 * slots + 8n = 192 KB there, embedding: 16n + 4 = 128 KB): opt in above 46 KB
  const int slots = tree_slots(n);
  const size_t tree_smem = (size_t)slots * 8 + (size_t)n * 8;
  static SmemOptIn tree_optin;
  if (tree_smem > 46 * 1024) GLOM_TRY(ln.check(tree_optin.ensure(island_tree_kernel, tree_smem)));
  island_tree_kernel<<<dim3(L, slabs), kTreeThreads, tree_smem, ln.st>>>(labels, n, slots, size, parent, containment,
                                                                          nested);
  GLOM_TRY(ln.launched());
  if (!states) return 0;
  const size_t embed_smem = ((size_t)n * 4 + 1) * 4;
  static SmemOptIn embed_optin;
  if (embed_smem > 46 * 1024) GLOM_TRY(ln.check(embed_optin.ensure(island_embed_kernel, embed_smem)));
  island_embed_kernel<<<dim3(L, slabs), kTreeThreads, embed_smem, ln.st>>>(labels, states, n, d, embedding, member_cos,
                                                                           coherence);
  return ln.launched();
}

}  // namespace glom
