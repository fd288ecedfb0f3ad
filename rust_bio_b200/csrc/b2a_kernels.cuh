// Small support kernels around K1/K2: K0 (pack/stage sequences into the
// TMA-friendly [task][word][pair] layout), ops compaction, and the fixed-stride
// result records that are all-gathered across GPUs.
#pragma once
#include <cuda_runtime.h>

#include "b2a_common.cuh"

namespace b2a {

struct PackParams {
  const Block* blocks;
  const uint32_t* order;    // sorted -> caller index
  const uint8_t* blob;      // caller's sequence blob (device copy)
  const uint64_t* x_off;    // caller order
  const uint32_t* x_len;
  const uint64_t* y_off;
  const uint32_t* y_len;
  const uint8_t* codemap;   // 256 bytes: symbol -> staged code (identity for MatchParams); 0xFF = not in alphabet
  uint8_t* seq;             // staged arena
  uint32_t* bad_symbol;     // set to 1 if a byte outside the alphabet is met
  int32_t G;
  int32_t mapped;           // codemap maps to LUT codes; 0: the identity map, where byte 0xFF is a symbol like any other
};

// K0: one CTA per block; each thread produces staged 32-bit words.
// Staged layout of a block (32-bit words): x: [task sub][word w][pair slot p], then y likewise,
// with P = 32/G pairs per task.  Bytes past the end of a sequence are 0.
__global__ void __launch_bounds__(256) pack_kernel(const PackParams prm) {
  __shared__ uint8_t cmap[256];  // symbol -> code, read four times per staged word
  __shared__ uint64_t s_off[64];  // the block's pairs: where x (0..31) and y (32..63) start in the blob ...
  __shared__ uint32_t s_len[64];  // ... and how long they are (one dependent chain per sequence, not per word)
  cmap[threadIdx.x] = prm.codemap[threadIdx.x];
  const Block blk = prm.blocks[blockIdx.x];
  if (threadIdx.x < 64) {
    const uint32_t pair = threadIdx.x & 31u;
    const bool isy = threadIdx.x >= 32;
    uint64_t off = 0;
    uint32_t len = 0;
    if (pair < blk.npairs) {
      const uint32_t orig = prm.order[blk.first + pair];
      off = isy ? prm.y_off[orig] : prm.x_off[orig];
      len = isy ? prm.y_len[orig] : prm.x_len[orig];
    }
    s_off[threadIdx.x] = off;
    s_len[threadIdx.x] = len;
  }
  __syncthreads();
  const int G = prm.G, P = 32 / G;
  uint32_t* out = reinterpret_cast<uint32_t*>(prm.seq + blk.seq_off);
  const uint32_t xtot = blk.xwords * 32, ytot = blk.ywords * 32;
  for (uint32_t k = threadIdx.x; k < xtot + ytot; k += blockDim.x) {
    const bool isy = k >= xtot;
    const uint32_t kk = isy ? k - xtot : k;
    const uint32_t words = isy ? blk.ywords : blk.xwords;
    // walk the pair fastest inside a sequence word so that a thread's 4 source bytes are adjacent
    const uint32_t pair = kk / words, w = kk % words;  // pair slot in block, word in sequence
    uint32_t val = 0;
    {
      const uint64_t off = s_off[pair + (isy ? 32u : 0u)];
      const uint32_t len = s_len[pair + (isy ? 32u : 0u)];  // 0 for the padding pairs of a last, partly filled block
      const uint32_t pos0 = w * 4;
      if (pos0 < len) {
        // the four source bytes in one load when the sequence starts on a word boundary and the word is whole
        uint32_t raw;
        const uint32_t have = len - pos0 < 4 ? len - pos0 : 4;
        if (((off & 3ull) == 0) && have == 4) {
          raw = *reinterpret_cast<const uint32_t*>(prm.blob + off + pos0);
        } else {
          raw = 0;
          for (uint32_t b = 0; b < have; ++b) raw |= (uint32_t)prm.blob[off + pos0 + b] << (8 * b);
        }
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          if ((uint32_t)b < have) {
            uint32_t code = cmap[(raw >> (8 * b)) & 0xFFu];
            if (prm.mapped && code == 0xFFu) {  // outside the scoring alphabet: flag it, stage a valid code
              *prm.bad_symbol = 1u;
              code = 0;
            }
            val |= code << (8 * b);
          }
        }
      }
    }
    const uint32_t sub = pair / P, p = pair % P;
    out[(isy ? (size_t)G * blk.xwords * P : 0) + ((size_t)sub * words + w) * P + p] = val;
  }
}

// which byte values occur in the blob (flags[v] != 0): decides the scoring alphabet
__global__ void __launch_bounds__(256) symbols_kernel(const uint8_t* __restrict__ blob, uint64_t n,
                                                      uint32_t* __restrict__ flags) {
  __shared__ uint32_t seen[256];
  seen[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += stride) seen[blob[i]] = 1u;
  __syncthreads();
  if (seen[threadIdx.x]) flags[threadIdx.x] = 1u;
}

// ops compaction: pair p's ops move from the walk scratch to ops_dense[ops_off[p] ..].
__global__ void gather_ops_kernel(const uint8_t* __restrict__ scratch,
                                  const uint64_t* __restrict__ ops_src,
                                  const uint64_t* __restrict__ ops_off, uint8_t* __restrict__ dense,
                                  uint64_t n_pairs) {
  const uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (warp >= n_pairs) return;
  const uint64_t lo = ops_off[warp], n = ops_off[warp + 1] - lo;
  const uint8_t* src = scratch + ops_src[warp];
  for (uint64_t k = lane; k < n; k += 32) dense[lo + k] = src[k];
}

// Small batches (n <= 65,536): exclusive sum of n_ops[0..n) into n+1 u64 offsets by ONE CTA with three barriers in
// all -- every 1,024-element round is warp-scanned up front (coalesced loads, the rounds are independent), the
// per-warp sums of every round are scanned by one warp each, the round totals by warp 0, and a second pass over the
// input adds the three levels up.  One launch instead of widen + the two passes of a device-wide scan.
__global__ void __launch_bounds__(1024) scan_small_kernel(const uint32_t* __restrict__ n_ops, uint64_t* __restrict__ off,
                                                          uint32_t n_pairs) {
  __shared__ uint32_t wsum[64][32];   // [round][warp]: inclusive warp totals, then exclusive within the round
  __shared__ uint32_t round_tot[64];
  __shared__ uint64_t round_base[65];
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  const uint32_t rounds = (n_pairs + 1023u) >> 10;  // <= 64
  auto warp_inc = [&](uint32_t v) {
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, v, d);
      if (lane >= (uint32_t)d) v += t;
    }
    return v;
  };
  for (uint32_t k = 0; k < rounds; ++k) {
    const uint32_t i = (k << 10) + threadIdx.x;
    const uint32_t inc = warp_inc(i < n_pairs ? n_ops[i] : 0u);  // a round's sum stays below 2^32: 1,024 x (m + n + 4) ops
    if (lane == 31) wsum[k][w] = inc;
  }
  __syncthreads();
  for (uint32_t k = w; k < rounds; k += 32) {
    const uint32_t ws = wsum[k][lane], wi = warp_inc(ws);
    wsum[k][lane] = wi - ws;
    if (lane == 31) round_tot[k] = wi;
  }
  __syncthreads();
  if (w == 0) {
    uint64_t carry = 0;
    for (uint32_t k0 = 0; k0 < rounds; k0 += 32) {
      const uint32_t k = k0 + lane;
      const uint64_t v = k < rounds ? (uint64_t)round_tot[k] : 0ull;
      uint64_t inc = v;
      for (int d = 1; d < 32; d <<= 1) {
        const uint64_t t = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= (uint32_t)d) inc += t;
      }
      if (k < rounds) round_base[k] = carry + inc - v;
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) round_base[rounds] = carry;
  }
  __syncthreads();
  for (uint32_t k = 0; k < rounds; ++k) {
    const uint32_t i = (k << 10) + threadIdx.x;
    const uint32_t v = i < n_pairs ? n_ops[i] : 0u;
    const uint32_t inc = warp_inc(v);
    if (i < n_pairs) off[i] = round_base[k] + wsum[k][w] + (inc - v);
  }
  if (threadIdx.x == 0) off[n_pairs] = round_base[rounds];
}

// n_ops (u32) -> u64 with a trailing 0 so one exclusive scan yields n_pairs+1 offsets
__global__ void widen_kernel(const uint32_t* __restrict__ n_ops, uint64_t* __restrict__ out,
                             uint64_t n_pairs) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i <= n_pairs) out[i] = i < n_pairs ? n_ops[i] : 0;
}

// fixed-stride records: {score, xstart, xend, ystart, yend, n_ops, clip_len[4]} + ops
__global__ void records_kernel(const int32_t* score, const uint32_t* xstart, const uint32_t* xend,
                               const uint32_t* ystart, const uint32_t* yend, const uint32_t* n_ops,
                               const uint32_t* clip_len, const uint8_t* scratch,
                               const uint64_t* ops_src, uint8_t* records, uint32_t stride,
                               uint64_t n_pairs) {
  const uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (warp >= n_pairs) return;
  uint8_t* rec = records + warp * stride;
  uint32_t* head = reinterpret_cast<uint32_t*>(rec);
  const uint32_t n = n_ops[warp];
  if (lane == 0) {
    head[0] = (uint32_t)score[warp];
    head[1] = xstart[warp];
    head[2] = xend[warp];
    head[3] = ystart[warp];
    head[4] = yend[warp];
    head[5] = n;
  }
  if (lane < 4) head[6 + lane] = clip_len[4 * warp + lane];
  const uint8_t* src = scratch + ops_src[warp];
  for (uint32_t k = lane; k < stride - 40; k += 32) rec[40 + k] = k < n ? src[k] : 0;
}

}  // namespace b2a
