// gn_partition.h -- how the persistent Gauss-Newton kernel (k_gn_loop, device_kernels.cuh) splits the moving leaves
// among its CTAs, and what the host reserves for that split.  One definition for both sides: the kernel takes its
// stretches from gn_stretch, and the launch sizes the per-CTA item map and the path memo from gn_share_bound, which
// bounds every share gn_stretch hands out.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "arith.h"

namespace madicp {

constexpr unsigned kGnPieces = 4;             // contiguous stretches of the moving leaves per CTA
constexpr size_t kGnMapMaxBytes = 16 * 1024;  // optional item map behind the staging tiles (GnArgs::map_in_smem)
constexpr unsigned kGnMapMaxLeaves = 1u << 26;  // the map packs an item as (keyframe << 26 | moving leaf)

// Stretch p (0 <= p < kGnPieces) of CTA b in a grid of G CTAs over L moving leaves: leaves [lo, lo + n).
// The leaves are cut into kGnPieces equal pieces and each piece into G stretches, dealt serpentine-wise (piece p of
// CTA b is stretch b for even p, stretch G-1-b for odd p): the cost of a stretch varies smoothly along the DFS order
// of the scan (tree depth, gate pass rate), so pairing opposite ends evens it out while every stretch stays one
// compact spatial region.  CTA 0 also folds the tiles of every round and solves: its stretches weigh 5 eighths of the
// others' (grids below 8 CTAs: equal weights), so that it is done with its own items early.  Over all CTAs the
// stretches of a piece tile it exactly once.
MADICP_HD void gn_stretch(unsigned L, unsigned G, unsigned b, unsigned p, unsigned& lo, unsigned& n) {
  const unsigned light = (G >= 8u) ? 3u : 0u;
  const uint64_t W8 = 8ull * G - light;                   // weight of a piece, in eighths of a share
  const unsigned s = (p & 1u) ? (G - 1u - b) : b;         // position of this CTA inside piece p
  const bool odd = (p & 1u) != 0u;
  // weight of the positions before `pos`: odd pieces put CTA 0 last, even pieces first
  const uint64_t c0 = odd ? 8ull * s : (s ? 8ull * s - light : 0ull);
  const uint64_t c1 = odd ? ((s + 1u >= G) ? W8 : 8ull * (s + 1u)) : 8ull * (s + 1u) - light;
  const uint64_t p0 = (uint64_t(L) * p) / kGnPieces, p1 = (uint64_t(L) * (p + 1u)) / kGnPieces;
  lo = unsigned(p0 + ((p1 - p0) * c0) / W8);
  n = unsigned(p0 + ((p1 - p0) * c1) / W8) - lo;
}

// An upper bound of every CTA's share (the sum of its kGnPieces stretches) that is monotone in L.  A stretch of weight
// w <= 8 in a piece of m leaves holds floor(p0 + m*c1/W8) - floor(p0 + m*c0/W8) < m*w/W8 + 1 leaves, and the pieces
// hold L leaves in all, so a share is < 8L/W8 + kGnPieces, i.e. <= ceil(8L/W8) + kGnPieces - 1.  It is exceeded by
// nobody and reached at some L (L = 429 716, G = 132: 3 268 leaves, 5 above floor(L/G) + 8).
MADICP_HD unsigned gn_share_bound(uint64_t L, unsigned G) {
  const uint64_t W8 = 8ull * G - ((G >= 8u) ? 3u : 0u);
  return unsigned((8ull * L + W8 - 1u) / W8) + kGnPieces - 1u;
}

// Bytes of the per-CTA item map for K keyframes: one 4-byte entry per CTA-local item, rounded up to whole warp groups
// (each warp writes 32 consecutive entries at a time), or 0 when the map does not fit in kGnMapMaxBytes or its
// packing.  The launch adds its own condition (the map must not move the CTA into the next carve-out).
MADICP_HD size_t gn_map_bytes(unsigned K, unsigned L, unsigned G) {
  if (L >= kGnMapMaxLeaves || K > 64u) return 0;
  const size_t entries = ((size_t(K) * gn_share_bound(L, G)) + 31u) & ~size_t(31);
  const size_t bytes = entries * 4u;
  return bytes <= kGnMapMaxBytes ? bytes : 0;
}

}  // namespace madicp
