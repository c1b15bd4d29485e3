// Host/device shared structures for the sm_90a attention kernels.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rfa {

constexpr int kDiagFull = 1 << 29;  // "no causal boundary": every key of the segment is visible

// One CTA work item: up to 128 consecutive query rows of one query chunk (two 64-row wgmma tiles).
struct alignas(16) WorkItem {
  int q_row0;     // first local query row
  int q_rows;     // 1..128
  int q_off;      // offset of q_row0 inside its chunk (the diagonal is expressed in chunk rows)
  int seg_begin;  // first entry in the segment table
  int seg_count;
  int pad0, pad1, pad2;
};

// A run of keys a chunk may see.  key j visible to chunk-row i  iff  j <= i + diag  and  j < kv_len.
struct alignas(16) KVSegment {
  int kv_row0;  // row inside the K/V tensor handed to this launch
  int kv_len;
  int diag;
  int flag;  // fused multi-GPU mode: index of the "rows have landed" flag to wait on, -1 = local data
};

// Tensor view handed to the launchers: (rows, heads, head_dim) with element strides.
struct TensorView {
  void* ptr;
  int64_t rows;
  int heads;
  int64_t row_stride;
  int64_t head_stride;
};

// ---- cross-GPU signalling (fused multi-GPU mode) ------------------------------------------------------
// Every rank owns a "signal pad" of uint32 epochs that its peers write over NVLink.
constexpr int kMaxRanks = 16;
constexpr int kPadKvReady = 0;      // [src]   src's K/V rows for me have landed in my staging buffer
constexpr int kPadConsumed = 64;    // [dst]   dst has finished reading what I pushed (staging reusable)
constexpr int kPadDkvReady = 128;   // [src]   src's dK/dV partials for my shard have landed in my inbox
constexpr int kPadInboxFree = 192;  // [owner] owner has reduced its inbox (I may overwrite my slot there)
constexpr int kPadWords = 1024;

// One contiguous run of K (or V) rows to copy from local memory into a peer's staging buffer.
// Offsets (not pointers) so that the table depends only on the plan and can be cached on the device.
struct alignas(16) PushTask {
  long long src_row;  // first local row of K (which == 0) or V (which == 1)
  long long dst_off;  // bytes from the destination's staging base (current parity) to the first staged row
  int rows;
  int dst;    // destination rank
  int which;  // 0 = K, 1 = V
  int pad;
};

// Plans that cannot derive their peers' plans locally (llama3: a rank only sees its own cu_seqlens slice) learn
// what every peer needs at run time: each rank's (source -> up to kNeedRanges row ranges) table is all-gathered
// on the device right before the launch and the push / reduce roles derive their work from it.
constexpr int kNeedRanges = 4;

struct PushParams {
  const PushTask* tasks;  // static mode: host-built table (plans that know their peers' plans)
  const int* dyn_needs;   // dynamic mode (tasks == nullptr): [dst][src][kNeedRanges][2] = (lo, hi) rows of src's shard
  int dyn_chunk_rows;     // rows per dynamic task
  int dyn_chunks;         // dynamic tasks per (destination, K|V, range)
  int world;
  long long region_bytes;  // bytes of the K half of one staging parity (V follows)
  int rows_cap;            // rows per source slot in the staging buffer
  int n_tasks;
  int n_ctas;     // blocks [0, n_ctas) of the grid are push CTAs
  int row_bytes;  // bytes per staged row (kv heads * 128 * 2)
  int my_rank;
  int use_tma;    // 1: bulk-copy (TMA) push, 0: LSU copy loop
  uint32_t epoch;
  long long parity_off;         // byte offset of the staging half used by this call
  const char* src_base[2];      // local K / V
  long long src_row_bytes[2];   // local row pitch of K / V
  char* stage_ptrs[kMaxRanks];  // peer-mapped staging base of every rank
  uint32_t* my_pad;
  uint32_t* peer_pads[kMaxRanks];
  uint32_t* sent_count;                // device counters, one per destination (cumulative)
  uint32_t sent_target[kMaxRanks];     // counter value that means "everything for this destination is out"
};

struct SignalParams {
  uint32_t* peer_pads[kMaxRanks];
  uint32_t* done_count;  // device counter (cumulative over calls)
  uint32_t done_target;
  uint32_t epoch;
  int world;    // 0 = signalling disabled
  int my_rank;
};

// Backward: where dK/dV tiles go.  owner slot o = (fp32 inbox of rank o, slot reserved for this rank).
struct DkvParams {
  void* dk_ptrs[kMaxRanks];  // owner o: this rank's slot in o's inbox (model dtype)
  void* dv_ptrs[kMaxRanks];
  uint32_t* peer_pads[kMaxRanks];
  uint32_t* my_pad;
  uint32_t* sent_count;               // device counters per owner (cumulative)
  uint32_t sent_target[kMaxRanks];
  uint32_t epoch;
  uint32_t wait_epoch;  // epoch of the previous backward call: owners must have reduced it before we overwrite
  int world;  // 0 = disabled: write to BwdParams::dk / dv
  int my_rank;
};

// Owner-side reduction of the inbox (model dtype partials, summed in fp32) into dK / dV (csrc/comm_sm90.cu).
struct alignas(16) ReduceTask {
  int row0, rows;
  unsigned src_mask;  // ranks whose slot holds a partial for these rows
  int pad;
};
struct ReduceParams {
  const ReduceTask* tasks;
  const int* dyn_needs;  // dynamic mode: the same all-gathered table (rows of MY shard that rank s returns = what it read)
  int n_tasks;
  const void* inbox;      // [world][2][rows_cap * hkv * 128], model dtype
  long long slot_stride;  // elements between slots
  long long kv_stride;    // elements between the dK and dV halves of a slot
  void* dk;               // (rows, hkv, 128) contiguous, output dtype
  void* dv;
  int row_elems;          // hkv * 128
  const uint32_t* my_pad;
  uint32_t* peer_pads[kMaxRanks];
  uint32_t* ticket;       // device counter (cumulative)
  uint32_t ticket_target;
  uint32_t epoch;
  int world, my_rank;
};
constexpr int kReduceBlocksPerTask = 128;
const char* reduce_dkv_launch(int dtype, const ReduceParams& p, cudaStream_t stream);
// out = cast(acc); acc = 0   (fp32 dQ accumulator -> model dtype, workspace left zeroed for the next backward)
const char* dq_finalize_launch(int dtype, float* acc, void* out, long long numel, cudaStream_t stream);

struct FwdParams {
  const WorkItem* items;
  const KVSegment* segs;
  const int* seg_lo;  // sliding window only (else nullptr): per segment, key j visible to chunk row i iff j >= i + lo
  // fp8 only: block descales.  q_scale[(row / q_scale_block) * hq + head]; k_scale / v_scale[(r / kv_scale_block) * hkv +
  // kv_head] with r = row in the K/V tensor the tile is read from (staging rows as they are; local rows + kv_scale_row0,
  // i.e. the tables cover [world][rows] in fused launches); v_ref[kv_head] = the head's largest V descale.
  const float* q_scale;
  const float* k_scale;
  const float* v_scale;
  const float* v_ref;
  int q_scale_block, kv_scale_block;
  long long kv_scale_row0;
  int flags;  // timing switches (RFA_B200_FWD_FLAGS): bit 1 = do not wait for remote K/V (compute-only timing,
              // wrong numbers); bit 2 = no compute (communication-only timing)
  void* out;  // (rows, hq, 128) contiguous, input dtype
  float* lse;  // index = (row / lse_S) * hq * lse_S + head * lse_S + row % lse_S
  int lse_S;
  int hq, hkv;
  int head_dim;      // 64 or 128 (selects the kernel instantiation)
  float scale;       // softmax scale
  float scale_log2;  // scale * log2(e)
  const uint32_t* ready_flags;  // fused mode only: this rank's signal pad (kPadKvReady + src)
  uint32_t ready_epoch;
  unsigned long long* trace;  // RFA_TRACE builds only: per-iteration clock64 stamps of CTA 0 (else unused)
  int n_items;       // compute CTAs = n_items * hq, laid out after the push CTAs
  PushParams push;   // n_ctas == 0 when there is nothing to push
  SignalParams sig;
};

// Backward work item: one tile of <= 128 keys (exclusive owner of those dK/dV rows in this launch).
struct alignas(16) BwdItem {
  int kv_row0;    // first row inside the K/V tensors handed to this launch
  int kv_rows;    // 1..128
  int seg_begin;  // first entry in the query-segment table
  int seg_count;
  int flag;  // fused mode: index of the "keys have landed" flag, -1 = local data
  int owner;     // fused mode: rank that owns these keys (selects the dK/dV destination)
  int out_row0;  // row of the tile inside the owner's shard (== kv_row0 when not fused)
  int pad2;
};
// A query chunk that can see the key tile.  tile key j visible to chunk row i  iff  i + lo <= j <= i + diag.
struct alignas(16) BwdQSegment {
  int q_row0;  // first local row of the chunk
  int q_len;
  int diag;  // already relative to the key tile's first key
  int lo;    // sliding-window launches only (BwdParams::window != 0), relative like diag; otherwise ignored
};

struct BwdParams {
  const BwdItem* items;
  const BwdQSegment* qsegs;
  const float* lse;    // same indexing as FwdParams::lse
  const float* delta;  // rowsum(out * dout), same indexing
  void* dk;            // (kv rows, hkv, 128), rows of each item are written (not accumulated); dtype: dkv_fp32
  void* dv;
  int dkv_fp32;        // 1: dk / dv are fp32 (fallback transports accumulate ring steps), 0: model dtype
  int lse_S;
  int hq, hkv;
  int head_dim;        // 64 or 128 (selects the kernel instantiation)
  float scale, scale_log2;
  const uint32_t* ready_flags;
  uint32_t ready_epoch;
  int n_items;
  int window;  // != 0: BwdQSegment::lo is meaningful (selects the kernel variant that masks the lower band edge)
  int item_major;  // CTA numbering: 0 = head-major (one GPU), 1 = key-tile-major (fused launches, table in ring order)
  int flags;       // timing switches (RFA_B200_BWD_FLAGS): bit 1 = do not wait for remote K/V, bit 2 = no compute
  unsigned long long* trace;  // RFA_TRACE builds only
  PushParams push;
  SignalParams sig;
  DkvParams dkv;
};

// dtype codes shared with the Python side
enum : int { kDtypeBF16 = 0, kDtypeFP16 = 1, kDtypeE4M3 = 2 };

// ---- launchers (implemented in the .cu files; plain C++ so bindings.cpp needs no CUDA headers beyond runtime)
// k_stage / v_stage: the peer-filled staging tensors read by segments with flag >= 0 (pass k / v when unused).
const char* attn_fwd_launch(int dtype, const TensorView& q, const TensorView& k, const TensorView& v,
                            const TensorView& k_stage, const TensorView& v_stage, const FwdParams& p,
                            cudaStream_t stream);

const char* attn_bwd_delta_launch(int dtype, const TensorView& out, const TensorView& dout, float* delta, int lse_S,
                                  int head_dim, cudaStream_t stream);
const char* attn_bwd_launch(int dtype, const TensorView& q, const TensorView& dout, const TensorView& k,
                            const TensorView& v, const TensorView& k_stage, const TensorView& v_stage,
                            const TensorView& dq_accum, const BwdParams& p, cudaStream_t stream);
const char* lse_flatten_launch(const float* in, float* out, const int* cu, int batch, int heads, int max_seqlen,
                               int total, cudaStream_t stream);
const char* lse_unflatten_launch(const float* in, float* out, const int* cu, int batch, int heads, int max_seqlen,
                                 cudaStream_t stream);
// Non-swizzled map with a (dim_inner, 1, box_rows) box (used for the fp32 dQ reduce-add).
const char* make_plain_tensor_map(CUtensorMap* out, const TensorView& t, int elem_bytes, int box_rows, int dim_inner);

// Encode a (rows, heads, 128) tensor as a 3-D TMA map with a (64, 1, box_rows) box and 128-byte swizzle.
// elem_bytes is 2 (bf16/fp16) or 4 (fp32; then the box is 32 elements wide) or 1 (e4m3: 128 elements).
// swizzle_bytes 64 selects the 64-byte swizzle and a box half as wide (e4m3 rows of 64 elements).
const char* make_tensor_map(CUtensorMap* out, const TensorView& t, int elem_bytes, int box_rows, int dim_inner,
                            int swizzle_bytes = 128);

}  // namespace rfa
