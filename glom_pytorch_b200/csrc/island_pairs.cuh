// Island pair counting shared by the part-whole trees (island_tree.cu: level l against level l + 1 of one slab) and the
// tracks (island_track.cu: slab t against slab t - 1 at one level).
//
// A patch i is a member of island j = lab[i] when 0 <= j <= i and lab[j] == j (include/glom_b200_tree.h); patches that
// fail are skipped, so garbage labels never index outside [0, n).  The pairs (j, k) of the islands one patch belongs to
// in two label maps are counted in a shared-memory hash table, one slot per distinct pair key j * n + k < 2^26:
//   slot = (key + 1) << 32 | count     (0 = empty; linear probing from mix(key); the table is never full)
// A sweep over the slots then hands each (j, k, count) to the caller, which keeps a maximum of pack_best keys:
//   pack_best(overlap, k) = overlap << 13 | (8191 - k)
// so the largest overlap wins and ties go to the smallest k whatever order the atomics land in.  overlap <= n <= 8192
// needs 14 bits, so a key fits in 27 bits; 0 means "no pair".
#pragma once

namespace glom {

constexpr int kKeyBits = 13;                      // k < n <= 8192 = 2^13
constexpr unsigned kKeyMask = (1u << kKeyBits) - 1;

// murmur3's 32-bit finaliser: pair keys j * n + k share their low bits for power-of-two n
__device__ __forceinline__ unsigned mix(unsigned h) {
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
  return h;
}

// the island patch i belongs to under the member rule above, or -1
__device__ __forceinline__ int member_of(const int* __restrict__ lab, int i) {
  const int j = lab[i];
  return (j >= 0 && j <= i && lab[j] == j) ? j : -1;
}

// hash-table slots of the pair table: a power of two >= 2n (load factor <= 1/2), at least 64
inline int tree_slots(int n) {
  int s = 64;
  while (s < 2 * n) s <<= 1;
  return s;
}

// count one patch in pair (j, k): key = j * n + k, mask = slots - 1
__device__ __forceinline__ void pair_insert(unsigned long long* table, unsigned mask, unsigned key) {
  const unsigned long long tag = (unsigned long long)(key + 1) << 32;
  for (unsigned h = mix(key) & mask;; h = (h + 1) & mask) {             // linear probing; never full
    const unsigned long long old = atomicCAS(&table[h], 0ull, tag | 1ull);
    if (old == 0ull) break;
    if ((old >> 32) == (unsigned long long)(key + 1)) { atomicAdd(&table[h], 1ull); break; }
  }
}

// every counted pair, once, spread over the block: f(j, k, overlap)
template <typename F>
__device__ __forceinline__ void pair_sweep(const unsigned long long* table, int slots, int n, F f) {
  for (int s = threadIdx.x; s < slots; s += blockDim.x) {
    const unsigned long long e = table[s];
    if (!e) continue;
    const unsigned key = (unsigned)(e >> 32) - 1, overlap = (unsigned)(e & 0xffffffffu);
    const unsigned j = key / (unsigned)n, k = key - j * (unsigned)n;
    f(j, k, overlap);
  }
}

__device__ __forceinline__ unsigned pack_best(unsigned overlap, unsigned k) { return overlap << kKeyBits | (kKeyMask - k); }
// the label of a pack_best maximum, or -1 for 0 (no pair)
__device__ __forceinline__ int best_label(unsigned b) { return b ? (int)(kKeyMask - (b & kKeyMask)) : -1; }
__device__ __forceinline__ int best_overlap(unsigned b) { return (int)(b >> kKeyBits); }

}  // namespace glom
