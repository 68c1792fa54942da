// me_cand.cuh — the kernel parameters of the candidate-list kernels, shared by me_cand.cu (the
// dispatcher and the grouped, warp and generic kernels) and me_chunk.cu (the staged chunk kernel).
#pragma once

#include "common.cuh"

namespace b200_me {

// Several (cur, ref) plane pairs served by one launch (me.rs:178-212 walks every allowed reference
// frame of every superblock; tiles and frames in flight add more): blocks, candidates and outputs
// are concatenated pair after pair, the table maps a block / group index back to its planes.
// Lives in the kernel parameters (constant bank, uniform lookups).
constexpr int kMaxPairs = 32;
struct MePairs {
  int n;
  uint32_t block_begin;            // first block of pair 0
  uint32_t block_end[kMaxPairs];   // pair k owns blocks [block_end[k-1], block_end[k])
  uint32_t group_end[kMaxPairs];   // grouped kernel: likewise for its groups (from 0)
  PlaneView cur[kMaxPairs], ref[kMaxPairs];
};

struct MeArgs {
  PlaneView cur, ref;  // == pr.cur[0] / pr.ref[0]; the only planes the generic kernels read
  const b200_block *blocks;
  const b200_cand *cands;
  const uint32_t *cand_offsets;  // CSR or null
  const short *pmv;              // 4 shorts per block (row0,col0,row1,col1) or null
  uint32_t *out_sad;
  unsigned long long *out_cost;
  b200_me_result *out_best;
  size_t ncands;
  size_t nblocks;
  int w, h;
  int w_in_b, h_in_b;
  uint32_t lambda;
  int allow_hp;
  int use_satd;
  int smem_bytes;  // dynamic smem given to the staged kernels
  size_t ngroups;  // ceil(nblocks / G) for the grouped kernel
  int hint_px;     // caller's bound on |mv|/8 (0 = unknown)
  // cooperative SAD kernel: every cost of the launch is below 2^27 - 1, so (cost << 5 | lane) is an
  // exact 32-bit warp key (launch_cand_group, from w, h, lambda and the largest rate)
  int key32;
  MePairs pr;
};

// me_chunk_lists (me_chunk.cu) for bpp, w x h and SAD / SATD over the pairs of `a`, or null where it
// has no instantiation: 8-bit SATD and 16-bit SAD / SATD, block sides multiples of 8, at most 32
// 8x8 chunks.
typedef int (*ChunkListsLaunch)(b200_ctx *ctx, const MeArgs &a);
ChunkListsLaunch chunk_lists_launcher(int bpp, int w, int h, bool satd);

}  // namespace b200_me
