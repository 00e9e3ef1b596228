// Counter-based dropout masks: keep(element index, site seed) is a pure function, so the backward pass regenerates
// the forward's mask instead of storing it.  (The reference uses torch's Philox stream, transformer.py:105,155,227;
// a fused kernel cannot reproduce that stream, so parity under dropout is statistical -- SURVEY.md section 7.)
//
// A site's seed derives from the per-call seed and the site's (layer, site) key.  The call seed is either a launch
// argument (the seed is derived on the host) or a device word read when the kernel runs (the seed is derived in the
// kernel): a CUDA graph that captures the launches then draws fresh masks on every replay once the word advances.
#pragma once
#include <cstdint>

namespace arb {

struct DropSite {
  uint32_t seed;      // per (call, layer, site) seed; unused when call_seed is set
  uint32_t thresh;    // drop iff hash < thresh  (thresh = p * 2^32); 0 disables the site
  float scale;        // 1 / (1 - p)
  uint32_t key;       // layer * 8 + site + 1: the site's part of the derivation (read with call_seed)
  const uint64_t* call_seed;   // null: use `seed`; else the call seed, read when the kernel runs (drop_seed)
};

__host__ __device__ __forceinline__ uint32_t mix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
  return h;
}
__host__ __device__ __forceinline__ bool drop_keep(unsigned long long idx, uint32_t seed, uint32_t thresh) {
  if (thresh == 0) return true;   // disabled site (may still carry a scale)
  uint32_t h = mix32(uint32_t(idx) ^ seed);
  h = mix32(h + uint32_t(idx >> 32) * 0x9e3779b1u + 0x7f4a7c15u);
  return h >= thresh;
}

// (call seed, site key) -> 32-bit site seed
__host__ __device__ __forceinline__ uint32_t site_seed(uint64_t call_seed, uint32_t key) {
  uint64_t z = call_seed + 0x9e3779b97f4a7c15ull * uint64_t(key);
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  z ^= z >> 31;
  return uint32_t(z) ^ uint32_t(z >> 32);
}

// The seed a kernel masks with.  A kernel calls this once per thread, before its element loops (and, when launched
// with PDL, after arb_pdl_wait(): the word may have been written by the kernel before it).
__device__ __forceinline__ uint32_t drop_seed(const DropSite& d) {
  return d.call_seed ? site_seed(*d.call_seed, d.key) : d.seed;
}

// The per-call seed: a host value, or (dev != null) a device word the kernels read when they execute
struct CallSeed {
  uint64_t value;
  const uint64_t* dev;
};

inline DropSite make_drop_site(CallSeed call, int layer, int site, float p) {
  DropSite d{0u, 0u, 1.0f};
  if (p <= 0.0f) return d;
  d.key = uint32_t(layer * 8 + site + 1);
  if (call.dev) d.call_seed = call.dev;
  else d.seed = site_seed(call.value, d.key);
  double t = double(p) * 4294967296.0;
  d.thresh = t >= 4294967295.0 ? 0xffffffffu : uint32_t(t);
  if (d.thresh == 0) d.thresh = 1;
  d.scale = 1.0f / (1.0f - p);
  return d;
}

enum { SITE_FC = 0, SITE_ATTN_P = 1, SITE_ATTN_OUT = 2, SITE_FFN_HID = 3, SITE_FFN_OUT = 4 };

}  // namespace arb
