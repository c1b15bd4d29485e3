// Host/device structures of the split-KV decode kernels (csrc/decode_sm90.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "attn_common.h"

namespace rfa {

// Partial results live in one fp32 buffer per split (or per rank): the (b, t, h) rows of `out` (rows x head_dim),
// followed by `lse` in the (b, h, t) order of the public softmax_lse.  part_stride = elements from one split's
// partial to the next, even for decode_kernel (it stores out as float2), so it may exceed the partial's size.  A varlen
// call (cu_seqlens_q set) uses the same layout at batch 1, sq = total_q: out rows (cu[b] + t, h), lse (h, cu[b] + t).
struct DecodeParams {
  const void* q;           // (B * Sq, Hq, D) view of (B, Sq, Hq, D), or varlen (total_q, Hq, D)
  long long q_row_stride;  // elements between consecutive (b, t)
  long long q_head_stride;
  const int* seqlens;      // (B,) valid cached rows of this rank's shard
  float* part;             // (n_splits, part_stride)
  long long part_stride;
  int batch, sq, hq, hkv;  // varlen: sq = max_seqlen_q, which bounds every count
  // Varlen queries: sequence b owns packed rows [cu[b], cu[b + 1]) of q, k_new / v_new and out; nullptr: every
  // sequence has sq rows, at b * sq.  Never validated: the kernels clamp every offset to [0, total_q] and every count
  // to [0, sq], so malformed values give an undefined result but no access outside the buffers.
  const int* cu_seqlens_q;  // (B + 1,)
  int total_q;              // rows of q: B * sq when uniform
  int s_cap;               // cache rows per sequence
  int tiles_per_split;     // 128-key tiles of one sequence handled by one split
  int n_new;               // nonzero iff keys are appended to this shard by this call (0 on all but the append rank)
  int causal;              // appended key u is visible to query token t only if u <= t
  float scale_log2;        // softmax scale * log2(e)
  // Paged caches: logical row j of sequence b is row j % page_size of page block_table[b * bt_stride + j / page_size]
  // of a pool of num_pages pages; the tensor maps then cover the (num_pages * page_size, Hkv, D) view of the pool.
  const int* block_table;  // nullptr when page_size == 0
  long long bt_stride;     // table entries between consecutive sequences
  int page_size;           // 0: contiguous (B, S_cap, Hkv, D) caches; else 16, 32, 64 or a multiple of 128
  int num_pages;
  // e4m3 caches: the cache holds x / descale, per (sequence, kv head); nullptr for bf16 / fp16 caches
  const float* k_descale;  // (B, Hkv) contiguous
  const float* v_descale;
  // Rotary embeddings of the new tokens; rotary_cos == nullptr: none.  Columns [0, 2 * rotary_half) of q and of the
  // appended k are rotated (pairs (i, i + rotary_half), or (2i, 2i + 1) when interleaved) at position
  // rotary_seqlens[b] + t for key t, and for query token t the same when causal, rotary_seqlens[b] otherwise (with a
  // tree mask: see tree_mask).
  // Positions are clamped to [0, seqlen_ro - 1], so a bad rotary_seqlens never reads outside the tables.
  const void* rotary_cos;    // (seqlen_ro, rotary_half) contiguous, in q's dtype
  const void* rotary_sin;
  const int* rotary_seqlens;  // (B,) first new token's position; read on the device only
  int rotary_half;            // rotary_dim / 2, a multiple of 8
  int seqlen_ro;
  int rotary_interleaved;
  // e4m3 queries (only over e4m3 caches): q holds x / q_descale[b, kv head]; nullptr for a bf16 / fp16 q
  const float* q_descale;  // (B, Hkv) contiguous; read on the device only
  // Contiguous caches only, both read on the device only.  Sequence b reads and appends slot cache_batch_idx[b] of a
  // (cache_batch, s_cap, Hkv, D) cache (nullptr: slot b); a slot outside [0, cache_batch) sees no key and drops its
  // append.  Its keys are rows [cache_leftpad[b], seqlens[b]) of the slot plus the appended rows (nullptr: from row
  // 0); the pad is clamped to [0, seqlens[b]].  Everything else (seqlens, descales, rotary) stays indexed by b.
  const int* cache_batch_idx;  // (B,)
  int cache_batch;
  const int* cache_leftpad;  // (B,)
  // Shared prefixes (decode_prefix_launch only): sequences [i * prefix_n, (i + 1) * prefix_n) share prefix i, whose
  // valid rows are seqlens[i] (clamped to [0, s_cap]) of a (P, s_cap, Hkv, D) cache, or with a block table of the
  // pages block_table[i * bt_stride + j] of a pool (the paged fields above, b = i); the descales are (P, Hkv).
  int prefix_n;
  // Tree attention (speculative decoding), with causal set; nullptr: none.  Byte u of row cu[b] + t (b * sq + t
  // uniform; row stride sq) is nonzero iff new token t of sequence b sees appended key u of its own call (u < n_b;
  // later columns are ignored).  It replaces the causal rule among the appended keys only: every cached key stays
  // visible.  New token t (query and key) is rotated at rotary_seqlens[b] + max(n_t - 1, 0), n_t = the nonzero
  // bytes of its row (a tree node's depth).  sq <= 128, so the appended keys span at most two key tiles.  Read on the
  // device only, never validated.
  const uint8_t* tree_mask;  // (total_q, sq)
};

// Appends k_new / v_new (B, Sq, Hkv, D), contiguous, in q's dtype, at rows [seqlens[b], seqlens[b] + Sq) of the
// caches (rows past the capacity, and with a block table rows whose page id is outside the pool, are dropped), then
// runs the split-KV kernel.  k_new == nullptr: attention only.  cache_dtype is dtype, or kDtypeE4M3 with
// p.k_descale / p.v_descale set: the append then stores e4m3(x / descale), saturated to +-448.  Varlen: k_new / v_new
// are (total_q, Hkv, D) and sequence b's n_b rows go to [seqlens[b], seqlens[b] + n_b); the grid is
// (n_splits, decode_tile_slots(p), Hkv), each slot mapped to a (sequence, row tile) on the device.  With
// p.rotary_cos set, q is rotated as the kernel loads it and k_new before it is stored (see DecodeParams).
// dtype is q's: kDtypeE4M3 (with p.q_descale) only over an e4m3 cache, where S = Q K^T is an e4m3 wgmma on the fp8
// K tile and the partials are those of a bf16 P V.  new_dtype is k_new / v_new's: q's, or kDtypeE4M3 over an e4m3
// cache (the bytes are stored as they are), or bf16 / fp16 with an e4m3 q.
const char* decode_fwd_launch(int dtype, int cache_dtype, const TensorView& k_cache, const TensorView& v_cache,
                              const void* k_new, const void* v_new, int new_dtype, const DecodeParams& p,
                              int n_splits, int head_dim, cudaStream_t stream);

// The shared-prefix pass: attention of every query row to its group's prefix, into the partial slabs of `p.part`
// (the same layout as decode_fwd_launch's; a caller merges both passes' slabs with one decode_combine_launch).  The
// caches k_prefix / v_prefix are (n_prefix, p.s_cap, Hkv, D) with mergeable first two dimensions, or with
// p.page_size set page pools (num_pages, page_size, Hkv, D) whose rows of prefix i are named by row i of p.block_table
// (p.s_cap = max_prefix_blocks * page_size; the same page sizes, boxes and skipped pages as decode_fwd_launch's paged
// cache); p.seqlens are the prefixes' valid rows, p.k_descale / p.v_descale (n_prefix, Hkv) with e4m3 caches,
// p.prefix_n = B / n_prefix.  Every prefix key is visible to every query token (p.n_new must be 0); q is rotated as
// in decode_fwd_launch (with p.tree_mask, at the depth positions; the mask does not mask prefix keys).  No append,
// cache slots, left pads or e4m3 q.  The grid is (n_splits, decode_prefix_slots(p), n_prefix *
// Hkv): a CTA takes 64 consecutive packed rows of one group, rows [b0 * sq, (b0 + n) * sq) of a uniform q or
// [cu[b0], cu[b0 + n]) of a varlen one (b0 = prefix * n), each row (sequence, token, head-in-group) in that order.
const char* decode_prefix_launch(int dtype, int cache_dtype, const TensorView& k_prefix, const TensorView& v_prefix,
                                 const DecodeParams& p, int n_prefix, int n_splits, int head_dim,
                                 cudaStream_t stream);

// Row-tile slots per (split, prefix, kv head) of the shared-prefix pass, from shapes only: ceil(rows * G / 64) for a
// group's rows, n * sq (uniform) or min(n * sq, total_q) (varlen, sq = max_seqlen_q).
long long decode_prefix_slots(const DecodeParams& p);

// Varlen row-tile slots, from shapes only: min(B * ceil(sq * G / 64), (total_q * G + 63 * B) / 64), an upper bound
// on sum_b ceil(n_b * G / 64) for any counts n_b <= sq that sum to total_q.
long long decode_tile_slots(const DecodeParams& p);

// Merges n_parts partials (part_stride elements apart) row by row in partial order.  out_dtype: kDtypeBF16,
// kDtypeFP16, or -1 for fp32.
const char* decode_combine_launch(const float* parts, long long part_stride, int n_parts, int batch, int sq, int hq,
                                  int head_dim, void* out, int out_dtype, float* lse, cudaStream_t stream);

}  // namespace rfa
