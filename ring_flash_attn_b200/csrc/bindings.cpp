// Python bindings for the sm_90a kernels and the peer-memory runtime (module ring_flash_attn_b200._C).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <cstdlib>

#include "attn_common.h"
#include "decode.h"
#include "peer_mem.h"

namespace {

using rfa::TensorView;

int dtype_code(const at::Tensor& t) {
  if (t.scalar_type() == at::kBFloat16) return rfa::kDtypeBF16;
  if (t.scalar_type() == at::kHalf) return rfa::kDtypeFP16;
  TORCH_CHECK(false, "ring_flash_attn_b200: only bf16 / fp16 inputs are supported by the sm_90a kernels");
}

TensorView view3(const at::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.dim() == 3, name, " must be (rows, heads, head_dim)");
  TORCH_CHECK(t.size(2) == 128 || t.size(2) == 64, name, ": the sm_90a kernels are instantiated for head_dim 64 and 128");
  TORCH_CHECK(t.stride(2) == 1, name, ": last dimension must be contiguous");
  return TensorView{t.data_ptr(), t.size(0), static_cast<int>(t.size(1)), t.stride(0), t.stride(1)};
}

void check(const char* err) { TORCH_CHECK(err == nullptr, "ring_flash_attn_b200 kernel launch failed: ", err); }

extern at::Tensor g_trace;

// Fused-mode context shared by the forward and backward launches (all lists are indexed by rank).
struct FusedCtx {
  at::Tensor k_stage, v_stage;   // (world * rows_cap, hkv, 128) views of this rank's staging buffer (current parity)
  at::Tensor my_pad;             // int32 view of this rank's signal pad
  at::Tensor push_tasks;         // int64 (n, 4); static mode
  c10::optional<at::Tensor> dyn_needs;  // int32 (world, world, kNeedRanges, 2): dynamic mode (llama3), see attn_common.h
  int64_t dyn_chunk_rows = 0, dyn_chunks = 0, rows_cap = 0, region_bytes = 0;
  at::Tensor counters;           // int32 (64): [0,16) kv sent, [16] done, [32,48) dkv sent, [48] reduce ticket
  std::vector<int64_t> stage_ptrs, pad_ptrs, sent_targets;
  int64_t n_push_ctas = 0, row_bytes = 0, my_rank = 0, world = 0, epoch = 0, done_target = 0, parity_off = 0;
  // backward only
  std::vector<int64_t> dk_ptrs, dv_ptrs, dkv_targets;
  int64_t dkv_wait_epoch = 0;
};

void fill_push(rfa::PushParams& pp, rfa::SignalParams& sg, const FusedCtx& c, const at::Tensor& k, const at::Tensor& v) {
  TORCH_CHECK(c.world <= rfa::kMaxRanks, "too many ranks for the fused path");
  TORCH_CHECK(c.push_tasks.scalar_type() == at::kLong && c.push_tasks.is_contiguous());
  TORCH_CHECK(k.stride(1) == k.size(2) && v.stride(1) == v.size(2),
              "K/V heads must be contiguous inside a row for the push path");
  uint32_t* cnt = reinterpret_cast<uint32_t*>(c.counters.data_ptr());
  pp.world = static_cast<int>(c.world);
  pp.rows_cap = static_cast<int>(c.rows_cap);
  pp.region_bytes = c.region_bytes;
  if (c.dyn_needs.has_value()) {
    const at::Tensor& nd = *c.dyn_needs;
    TORCH_CHECK(nd.scalar_type() == at::kInt && nd.is_cuda() && nd.is_contiguous() &&
                nd.numel() == c.world * c.world * rfa::kNeedRanges * 2, "dyn_needs: int32 (world, world, ranges, 2)");
    pp.tasks = nullptr;
    pp.dyn_needs = nd.data_ptr<int>();
    pp.dyn_chunk_rows = static_cast<int>(c.dyn_chunk_rows);
    pp.dyn_chunks = static_cast<int>(c.dyn_chunks);
    pp.n_tasks = static_cast<int>((c.world - 1) * 2 * rfa::kNeedRanges * c.dyn_chunks);
  } else {
    pp.tasks = reinterpret_cast<const rfa::PushTask*>(c.push_tasks.data_ptr());
    pp.n_tasks = static_cast<int>(c.push_tasks.size(0));
  }
  pp.n_ctas = pp.n_tasks > 0 ? static_cast<int>(c.n_push_ctas) : 0;
  pp.row_bytes = static_cast<int>(c.row_bytes);
  pp.my_rank = static_cast<int>(c.my_rank);
  {
    const char* e = std::getenv("RFA_B200_PUSH_TMA");
    pp.use_tma = e ? std::atoi(e) : 1;
    // bulk copies need 16-byte aligned rows on both sides
    if ((c.row_bytes % 16) || ((k.stride(0) * k.element_size()) % 16) || ((v.stride(0) * v.element_size()) % 16)) pp.use_tma = 0;
  }
  pp.epoch = static_cast<uint32_t>(c.epoch);
  pp.parity_off = c.parity_off;
  pp.src_base[0] = static_cast<const char*>(k.data_ptr());
  pp.src_base[1] = static_cast<const char*>(v.data_ptr());
  pp.src_row_bytes[0] = k.stride(0) * k.element_size();
  pp.src_row_bytes[1] = v.stride(0) * v.element_size();
  pp.my_pad = reinterpret_cast<uint32_t*>(c.my_pad.data_ptr());
  pp.sent_count = cnt;
  sg.done_count = cnt + 16;
  sg.done_target = static_cast<uint32_t>(c.done_target);
  sg.epoch = static_cast<uint32_t>(c.epoch);
  sg.world = static_cast<int>(c.world);
  sg.my_rank = static_cast<int>(c.my_rank);
  for (int r = 0; r < c.world; ++r) {
    pp.stage_ptrs[r] = reinterpret_cast<char*>(c.stage_ptrs[r]);
    pp.peer_pads[r] = reinterpret_cast<uint32_t*>(c.pad_ptrs[r]);
    pp.sent_target[r] = static_cast<uint32_t>(c.sent_targets[r]);
    sg.peer_pads[r] = reinterpret_cast<uint32_t*>(c.pad_ptrs[r]);
  }
}

// Block descales of the fp8 forward (see FwdParams): tables are (blocks, heads) fp32.
struct Fp8Scales {
  at::Tensor q, k, v, v_ref;
  int64_t q_block = 1, kv_block = 128, kv_row0 = 0;
};

void attn_fwd_impl(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, const at::Tensor& items,
                   const at::Tensor& segs, at::Tensor& out, at::Tensor& lse, int64_t lse_S, double scale,
                   const FusedCtx* fc, const at::Tensor* seg_lo = nullptr, const Fp8Scales* f8 = nullptr) {
  const c10::cuda::CUDAGuard guard(q.device());
  const bool fp8 = f8 != nullptr;
  TORCH_CHECK(items.scalar_type() == at::kInt && items.is_cuda() && items.is_contiguous() && items.size(1) == 8);
  TORCH_CHECK(segs.scalar_type() == at::kInt && segs.is_cuda() && segs.is_contiguous() && segs.size(1) == 4);
  TORCH_CHECK(out.is_contiguous() && out.scalar_type() == (fp8 ? at::kBFloat16 : q.scalar_type()));
  TORCH_CHECK(lse.is_contiguous() && lse.scalar_type() == at::kFloat);
  TORCH_CHECK(k.scalar_type() == q.scalar_type() && v.scalar_type() == q.scalar_type());
  TORCH_CHECK(q.size(1) % k.size(1) == 0, "query heads must be a multiple of kv heads");
  rfa::FwdParams p{};
  p.items = reinterpret_cast<const rfa::WorkItem*>(items.data_ptr());
  p.segs = reinterpret_cast<const rfa::KVSegment*>(segs.data_ptr());
  if (seg_lo != nullptr) {
    TORCH_CHECK(seg_lo->scalar_type() == at::kInt && seg_lo->is_cuda() && seg_lo->is_contiguous() &&
                seg_lo->numel() == segs.size(0), "seg_lo must hold one int32 per segment");
    p.seg_lo = seg_lo->data_ptr<int>();
  }
  int dtype = 0;
  if (fp8) {
    TORCH_CHECK(q.scalar_type() == at::kFloat8_e4m3fn, "the fp8 forward takes float8_e4m3fn q / k / v");
    auto table = [&](const at::Tensor& t, int64_t heads, const char* name) {
      TORCH_CHECK(t.scalar_type() == at::kFloat && t.is_cuda() && t.is_contiguous() && t.dim() == 2 &&
                  t.size(1) == heads && t.size(0) >= 1, name, ": fp32 (blocks, heads) descale table");
      return t.data_ptr<float>();
    };
    p.q_scale = table(f8->q, q.size(1), "q_scale");
    p.k_scale = table(f8->k, k.size(1), "k_scale");
    p.v_scale = table(f8->v, k.size(1), "v_scale");
    TORCH_CHECK(f8->v_ref.scalar_type() == at::kFloat && f8->v_ref.is_cuda() && f8->v_ref.is_contiguous() &&
                f8->v_ref.numel() == k.size(1), "v_ref: one fp32 per kv head");
    TORCH_CHECK(f8->k.size(0) == f8->v.size(0), "k_scale / v_scale must have the same number of blocks");
    p.v_ref = f8->v_ref.data_ptr<float>();
    TORCH_CHECK(f8->q_block >= 1 && f8->q.size(0) * f8->q_block >= q.size(0), "q_scale does not cover the query rows");
    TORCH_CHECK(f8->kv_block >= 1 && (f8->kv_block % 128 == 0 || f8->k.size(0) == 1),
                "k / v descale blocks must be multiples of 128 rows (one scale per key tile) or one per head");
    p.q_scale_block = static_cast<int>(f8->q_block);
    p.kv_scale_block = static_cast<int>(f8->kv_block);
    p.kv_scale_row0 = f8->kv_row0;
    dtype = rfa::kDtypeE4M3;
  } else {
    dtype = dtype_code(q);
  }
  p.out = out.data_ptr();
  p.lse = lse.data_ptr<float>();
  p.lse_S = static_cast<int>(lse_S);
  p.hq = static_cast<int>(q.size(1));
  p.hkv = static_cast<int>(k.size(1));
  p.head_dim = static_cast<int>(q.size(2));
  TORCH_CHECK(k.size(2) == q.size(2) && v.size(2) == q.size(2) && out.size(2) == q.size(2), "head_dim mismatch");
  p.scale = static_cast<float>(scale);
  p.scale_log2 = static_cast<float>(scale * 1.4426950408889634);
  p.n_items = static_cast<int>(items.size(0));
  p.trace = g_trace.defined() ? reinterpret_cast<unsigned long long*>(g_trace.data_ptr()) : nullptr;
  auto* launch_fwd = &rfa::attn_fwd_launch;
  {
    static const int fwd_flags = [] {
      const char* e = std::getenv("RFA_B200_FWD_FLAGS");
      return e ? std::atoi(e) : 0;
    }();
    p.flags = fwd_flags;
  }
  if (fc != nullptr) {
    p.ready_flags = reinterpret_cast<const uint32_t*>(fc->my_pad.data_ptr()) + rfa::kPadKvReady;
    p.ready_epoch = static_cast<uint32_t>(fc->epoch);
    fill_push(p.push, p.sig, *fc, k, v);
    check(launch_fwd(dtype, view3(q, "q"), view3(k, "k"), view3(v, "v"),
                               view3(fc->k_stage, "k_stage"), view3(fc->v_stage, "v_stage"), p,
                               at::cuda::getCurrentCUDAStream()));
  } else {
    check(launch_fwd(dtype, view3(q, "q"), view3(k, "k"), view3(v, "v"), view3(k, "k"), view3(v, "v"), p,
                     at::cuda::getCurrentCUDAStream()));
  }
}

at::Tensor g_trace;  // optional clock64 trace buffer (RFA_TRACE builds)

void set_trace(const c10::optional<at::Tensor>& t) { g_trace = t.has_value() ? *t : at::Tensor(); }

void attn_fwd(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, const at::Tensor& items,
              const at::Tensor& segs, at::Tensor& out, at::Tensor& lse, int64_t lse_S, double scale) {
  attn_fwd_impl(q, k, v, items, segs, out, lse, lse_S, scale, nullptr);
}

// fp8 forward: q / k / v float8_e4m3fn (rows, heads, 128), out bf16, block descales:
//   q_scale (ceil(rows / q_block), Hq), k_scale / v_scale (blocks of kv_block rows, Hkv), v_ref (Hkv) = max of v_scale
//   per head; kv_row0 = row of local key row 0 inside the k / v scale tables.
void attn_fwd_fp8(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, const at::Tensor& items,
                  const at::Tensor& segs, const at::Tensor& q_scale, int64_t q_block, const at::Tensor& k_scale,
                  const at::Tensor& v_scale, int64_t kv_block, const at::Tensor& v_ref, int64_t kv_row0,
                  at::Tensor& out, at::Tensor& lse, int64_t lse_S, double scale) {
  Fp8Scales f8{q_scale, k_scale, v_scale, v_ref, q_block, kv_block, kv_row0};
  attn_fwd_impl(q, k, v, items, segs, out, lse, lse_S, scale, nullptr, nullptr, &f8);
}

// The same inside the fused multi-GPU launch (K/V rows travel as one byte per element; the k / v tables cover
// [world][rows] like the staging buffer).
void attn_fwd_fused_fp8(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, const at::Tensor& items,
                        const at::Tensor& segs, const at::Tensor& q_scale, int64_t q_block, const at::Tensor& k_scale,
                        const at::Tensor& v_scale, int64_t kv_block, const at::Tensor& v_ref, int64_t kv_row0,
                        at::Tensor& out, at::Tensor& lse, int64_t lse_S, double scale, const FusedCtx& fc) {
  Fp8Scales f8{q_scale, k_scale, v_scale, v_ref, q_block, kv_block, kv_row0};
  attn_fwd_impl(q, k, v, items, segs, out, lse, lse_S, scale, &fc, nullptr, &f8);
}

// Sliding-window launch: seg_lo[i] is the lower band offset of segment i (see FwdParams::seg_lo).
void attn_fwd_window(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, const at::Tensor& items,
                     const at::Tensor& segs, const at::Tensor& seg_lo, at::Tensor& out, at::Tensor& lse, int64_t lse_S,
                     double scale) {
  attn_fwd_impl(q, k, v, items, segs, out, lse, lse_S, scale, nullptr, &seg_lo);
}

void attn_fwd_fused(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, const at::Tensor& items,
                    const at::Tensor& segs, at::Tensor& out, at::Tensor& lse, int64_t lse_S, double scale,
                    const FusedCtx& fc) {
  attn_fwd_impl(q, k, v, items, segs, out, lse, lse_S, scale, &fc);
}

void attn_fwd_fused_window(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, const at::Tensor& items,
                           const at::Tensor& segs, const at::Tensor& seg_lo, at::Tensor& out, at::Tensor& lse,
                           int64_t lse_S, double scale, const FusedCtx& fc) {
  attn_fwd_impl(q, k, v, items, segs, out, lse, lse_S, scale, &fc, &seg_lo);
}

void attn_bwd_delta(const at::Tensor& out, const at::Tensor& dout, at::Tensor& delta, int64_t lse_S) {
  const c10::cuda::CUDAGuard guard(out.device());
  TORCH_CHECK(delta.is_contiguous() && delta.scalar_type() == at::kFloat);
  check(rfa::attn_bwd_delta_launch(dtype_code(out), view3(out, "out"), view3(dout, "dout"), delta.data_ptr<float>(),
                                   static_cast<int>(lse_S), static_cast<int>(out.size(2)),
                                   at::cuda::getCurrentCUDAStream()));
}

void attn_bwd_impl(const at::Tensor& q, const at::Tensor& dout, const at::Tensor& k, const at::Tensor& v,
                   at::Tensor& dq_accum, const at::Tensor& items, const at::Tensor& qsegs, const at::Tensor& lse,
                   const at::Tensor& delta, const c10::optional<at::Tensor>& dk, const c10::optional<at::Tensor>& dv,
                   int64_t lse_S, double scale, const FusedCtx* fc, bool window = false) {
  const c10::cuda::CUDAGuard guard(q.device());
  TORCH_CHECK(items.scalar_type() == at::kInt && items.is_cuda() && items.is_contiguous() && items.size(1) == 8);
  TORCH_CHECK(qsegs.scalar_type() == at::kInt && qsegs.is_cuda() && qsegs.is_contiguous() && qsegs.size(1) == 4);
  TORCH_CHECK(dq_accum.scalar_type() == at::kFloat && dq_accum.dim() == 3 && dq_accum.size(2) == q.size(2) &&
              dq_accum.stride(2) == 1);
  if (fc == nullptr) {
    TORCH_CHECK(dk.has_value() && dv.has_value());
    TORCH_CHECK(dk->is_contiguous() && dv->is_contiguous() && dk->scalar_type() == dv->scalar_type());
    TORCH_CHECK(dk->scalar_type() == at::kFloat || dk->scalar_type() == q.scalar_type(),
                "dk / dv must be fp32 (accumulating transports) or the model dtype");
  }
  TORCH_CHECK(lse.scalar_type() == at::kFloat && delta.scalar_type() == at::kFloat);
  rfa::BwdParams p{};
  p.items = reinterpret_cast<const rfa::BwdItem*>(items.data_ptr());
  p.qsegs = reinterpret_cast<const rfa::BwdQSegment*>(qsegs.data_ptr());
  p.lse = lse.data_ptr<float>();
  p.delta = delta.data_ptr<float>();
  p.dk = dk.has_value() ? dk->data_ptr() : nullptr;
  p.dv = dv.has_value() ? dv->data_ptr() : nullptr;
  p.dkv_fp32 = (dk.has_value() && dk->scalar_type() == at::kFloat) ? 1 : 0;
  p.lse_S = static_cast<int>(lse_S);
  p.hq = static_cast<int>(q.size(1));
  p.hkv = static_cast<int>(k.size(1));
  p.head_dim = static_cast<int>(q.size(2));
  p.scale = static_cast<float>(scale);
  p.scale_log2 = static_cast<float>(scale * 1.4426950408889634);
  TensorView dqv{dq_accum.data_ptr(), dq_accum.size(0), static_cast<int>(dq_accum.size(1)), dq_accum.stride(0),
                 dq_accum.stride(1)};
  p.n_items = static_cast<int>(items.size(0));
  p.window = window ? 1 : 0;
  p.trace = g_trace.defined() ? reinterpret_cast<unsigned long long*>(g_trace.data_ptr()) : nullptr;
  if (fc != nullptr) {
    p.ready_flags = reinterpret_cast<const uint32_t*>(fc->my_pad.data_ptr()) + rfa::kPadKvReady;
    p.ready_epoch = static_cast<uint32_t>(fc->epoch);
    fill_push(p.push, p.sig, *fc, k, v);
    uint32_t* cnt = reinterpret_cast<uint32_t*>(fc->counters.data_ptr());
    {
      static const int item_major = [] {
        const char* e = std::getenv("RFA_B200_BWD_TILE_MAJOR");
        return e ? std::atoi(e) : 1;
      }();
      p.item_major = item_major;
      static const int bwd_flags = [] {
        const char* e = std::getenv("RFA_B200_BWD_FLAGS");
        return e ? std::atoi(e) : 0;
      }();
      p.flags = bwd_flags;
    }
    p.dkv.my_pad = reinterpret_cast<uint32_t*>(fc->my_pad.data_ptr());
    p.dkv.sent_count = cnt + 32;
    p.dkv.epoch = static_cast<uint32_t>(fc->epoch);
    p.dkv.wait_epoch = static_cast<uint32_t>(fc->dkv_wait_epoch);
    p.dkv.world = static_cast<int>(fc->world);
    p.dkv.my_rank = static_cast<int>(fc->my_rank);
    for (int r = 0; r < fc->world; ++r) {
      p.dkv.dk_ptrs[r] = reinterpret_cast<void*>(fc->dk_ptrs[r]);
      p.dkv.dv_ptrs[r] = reinterpret_cast<void*>(fc->dv_ptrs[r]);
      p.dkv.peer_pads[r] = reinterpret_cast<uint32_t*>(fc->pad_ptrs[r]);
      p.dkv.sent_target[r] = static_cast<uint32_t>(fc->dkv_targets[r]);
    }
    check(rfa::attn_bwd_launch(dtype_code(q), view3(q, "q"), view3(dout, "dout"), view3(k, "k"), view3(v, "v"),
                               view3(fc->k_stage, "k_stage"), view3(fc->v_stage, "v_stage"), dqv, p,
                               at::cuda::getCurrentCUDAStream()));
  } else {
    check(rfa::attn_bwd_launch(dtype_code(q), view3(q, "q"), view3(dout, "dout"), view3(k, "k"), view3(v, "v"),
                               view3(k, "k"), view3(v, "v"), dqv, p, at::cuda::getCurrentCUDAStream()));
  }
}

void attn_bwd(const at::Tensor& q, const at::Tensor& dout, const at::Tensor& k, const at::Tensor& v,
              at::Tensor& dq_accum, const at::Tensor& items, const at::Tensor& qsegs, const at::Tensor& lse,
              const at::Tensor& delta, at::Tensor& dk, at::Tensor& dv, int64_t lse_S, double scale) {
  attn_bwd_impl(q, dout, k, v, dq_accum, items, qsegs, lse, delta, dk, dv, lse_S, scale, nullptr);
}

// Sliding-window launch: column 3 of qsegs carries the lower band offset (BwdQSegment::lo).
void attn_bwd_window(const at::Tensor& q, const at::Tensor& dout, const at::Tensor& k, const at::Tensor& v,
                     at::Tensor& dq_accum, const at::Tensor& items, const at::Tensor& qsegs, const at::Tensor& lse,
                     const at::Tensor& delta, at::Tensor& dk, at::Tensor& dv, int64_t lse_S, double scale) {
  attn_bwd_impl(q, dout, k, v, dq_accum, items, qsegs, lse, delta, dk, dv, lse_S, scale, nullptr, true);
}

void attn_bwd_fused(const at::Tensor& q, const at::Tensor& dout, const at::Tensor& k, const at::Tensor& v,
                    at::Tensor& dq_accum, const at::Tensor& items, const at::Tensor& qsegs, const at::Tensor& lse,
                    const at::Tensor& delta, int64_t lse_S, double scale, const FusedCtx& fc) {
  attn_bwd_impl(q, dout, k, v, dq_accum, items, qsegs, lse, delta, c10::nullopt, c10::nullopt, lse_S, scale, &fc);
}

void attn_bwd_fused_window(const at::Tensor& q, const at::Tensor& dout, const at::Tensor& k, const at::Tensor& v,
                           at::Tensor& dq_accum, const at::Tensor& items, const at::Tensor& qsegs,
                           const at::Tensor& lse, const at::Tensor& delta, int64_t lse_S, double scale,
                           const FusedCtx& fc) {
  attn_bwd_impl(q, dout, k, v, dq_accum, items, qsegs, lse, delta, c10::nullopt, c10::nullopt, lse_S, scale, &fc,
                true);
}

// Owner-side reduction of the dK/dV inbox (csrc/comm_sm90.cu).
void reduce_dkv(const at::Tensor& inbox, int64_t slot_stride, int64_t kv_stride, at::Tensor& dk, at::Tensor& dv,
                const at::Tensor& tasks, const FusedCtx& fc, int64_t ticket_target) {
  const c10::cuda::CUDAGuard guard(inbox.device());
  TORCH_CHECK(inbox.scalar_type() == dk.scalar_type() && dk.is_contiguous() && dv.is_contiguous());
  TORCH_CHECK(tasks.scalar_type() == at::kInt && tasks.is_contiguous() && tasks.size(1) == 4);
  rfa::ReduceParams p{};
  p.tasks = reinterpret_cast<const rfa::ReduceTask*>(tasks.data_ptr());
  p.n_tasks = static_cast<int>(tasks.size(0));
  p.dyn_needs = fc.dyn_needs.has_value() ? fc.dyn_needs->data_ptr<int>() : nullptr;
  p.inbox = inbox.data_ptr();
  p.slot_stride = slot_stride;
  p.kv_stride = kv_stride;
  p.dk = dk.data_ptr();
  p.dv = dv.data_ptr();
  p.row_elems = static_cast<int>(dk.size(1) * dk.size(2));
  p.my_pad = reinterpret_cast<const uint32_t*>(fc.my_pad.data_ptr());
  p.ticket = reinterpret_cast<uint32_t*>(fc.counters.data_ptr()) + 48;
  p.ticket_target = static_cast<uint32_t>(ticket_target);
  p.epoch = static_cast<uint32_t>(fc.epoch);
  p.world = static_cast<int>(fc.world);
  p.my_rank = static_cast<int>(fc.my_rank);
  for (int r = 0; r < fc.world; ++r) p.peer_pads[r] = reinterpret_cast<uint32_t*>(fc.pad_ptrs[r]);
  check(rfa::reduce_dkv_launch(dtype_code(dk), p, at::cuda::getCurrentCUDAStream()));
}

// dq = cast(acc); acc = 0  (csrc/comm_sm90.cu: dq_finalize_kernel)
void dq_finalize(at::Tensor& acc, at::Tensor& out) {
  const c10::cuda::CUDAGuard guard(acc.device());
  TORCH_CHECK(acc.scalar_type() == at::kFloat && acc.is_contiguous() && out.is_contiguous() &&
              acc.numel() == out.numel());
  check(rfa::dq_finalize_launch(dtype_code(out), acc.data_ptr<float>(), out.data_ptr(), acc.numel(),
                                at::cuda::getCurrentCUDAStream()));
}

at::Tensor lse_flatten(const at::Tensor& lse, const at::Tensor& cu) {
  const c10::cuda::CUDAGuard guard(lse.device());
  TORCH_CHECK(lse.dim() == 3 && lse.scalar_type() == at::kFloat && lse.is_contiguous());
  TORCH_CHECK(cu.scalar_type() == at::kInt && cu.is_cuda());
  const int batch = static_cast<int>(cu.numel()) - 1;
  const int64_t total = cu[batch].item<int>();
  at::Tensor out = at::empty({lse.size(1), total}, lse.options());
  check(rfa::lse_flatten_launch(lse.data_ptr<float>(), out.data_ptr<float>(), cu.data_ptr<int>(), batch,
                                static_cast<int>(lse.size(1)), static_cast<int>(lse.size(2)), static_cast<int>(total),
                                at::cuda::getCurrentCUDAStream()));
  return out;
}

at::Tensor lse_unflatten(const at::Tensor& lse, const at::Tensor& cu, int64_t max_seqlen) {
  const c10::cuda::CUDAGuard guard(lse.device());
  TORCH_CHECK(lse.dim() == 3 && lse.size(2) == 1 && lse.scalar_type() == at::kFloat && lse.is_contiguous());
  TORCH_CHECK(cu.scalar_type() == at::kInt && cu.is_cuda());
  const int batch = static_cast<int>(cu.numel()) - 1;
  at::Tensor out = at::empty({batch, lse.size(1), max_seqlen}, lse.options());
  check(rfa::lse_unflatten_launch(lse.data_ptr<float>(), out.data_ptr<float>(), cu.data_ptr<int>(), batch,
                                  static_cast<int>(lse.size(1)), static_cast<int>(max_seqlen),
                                  at::cuda::getCurrentCUDAStream()));
  return out;
}

// A tree mask of decode_fwd / decode_prefix_fwd: bool or uint8 (rows, sq) contiguous on q's device, with causal.
const uint8_t* tree_mask_ptr(const c10::optional<at::Tensor>& tree_mask, const at::Tensor& q, int64_t rows,
                             int64_t sq, bool causal, const char* what) {
  if (!tree_mask.has_value()) return nullptr;
  const at::Tensor& m = *tree_mask;
  TORCH_CHECK(m.scalar_type() == at::kBool || m.scalar_type() == at::kByte, what,
              ": tree_mask must be bool or uint8");
  TORCH_CHECK(m.device() == q.device() && m.is_contiguous() && m.dim() == 2 && m.size(0) == rows && m.size(1) == sq,
              what, ": tree_mask must be contiguous (B * Sq, Sq), or (total_q, max_seqlen_q) when varlen, on q's "
              "device");
  TORCH_CHECK(causal, what, ": a tree mask replaces the causal rule among the appended keys: it needs causal");
  TORCH_CHECK(sq <= 128, what, ": a tree mask takes at most 128 new tokens per sequence (two key tiles)");
  return static_cast<const uint8_t*>(m.data_ptr());
}

// Split-KV decode (csrc/decode_sm90.cu).  q (B, Sq, Hq, D); k_cache / v_cache (B, S_cap, Hkv, D) with mergeable
// batch and sequence dimensions; seqlens (B,) int32; k_new / v_new (B, Sq, Hkv, D) contiguous, appended to the caches
// before attention when given.  part: fp32 (n_splits, B*Sq*Hq*D + B*Hq*Sq), see DecodeParams.  With block_table
// (B, max_blocks) int32, the caches are page pools (num_blocks, page_size, Hkv, D) with mergeable page and row
// dimensions, and S_cap = max_blocks * page_size.  The caches may instead both be float8_e4m3fn, with k_descale /
// v_descale fp32 (B, Hkv) contiguous on q's device: the cache then holds x / descale[b, kv head].  With cu_seqlens_q
// (B + 1,) int32 (B = seqlens.numel()), q is varlen (total_q, Hq, D), k_new / v_new (total_q, Hkv, D), part fp32
// (n_splits, total_q*Hq*D + Hq*total_q), and max_seqlen_q >= 1 bounds every count; cu_seqlens_q is not validated.
// With rotary_cos / rotary_sin (seqlen_ro, rotary_dim / 2) contiguous in q's dtype and rotary_seqlens (B,) int32,
// q and the appended k are rotated (see DecodeParams); rotary_seqlens is read on the device only.  q may be
// float8_e4m3fn over e4m3 caches, with q_descale fp32 (B, Hkv) contiguous on q's device (partials of a bf16 P V);
// k_new / v_new may be float8_e4m3fn over e4m3 caches (stored as they are), or bf16 / fp16 with an e4m3 q.
// cache_batch_idx (B,) int32 (contiguous caches only): sequence b reads and appends slot cache_batch_idx[b] of
// (B_cache, S_cap, Hkv, D) caches; cache_leftpad (B,) int32: its keys start at that row.  Both are read on the device
// only (see DecodeParams).  tree_mask (B * Sq, Sq), or (total_q, max_seqlen_q) when varlen, bool / uint8, with
// causal: which appended keys each new token sees, and the rotary positions (see DecodeParams); read on the device
// only.
void decode_fwd(const at::Tensor& q_in, at::Tensor& k_cache, at::Tensor& v_cache, const at::Tensor& seqlens,
                const c10::optional<at::Tensor>& k_new, const c10::optional<at::Tensor>& v_new, bool causal,
                double scale, at::Tensor& part, const c10::optional<at::Tensor>& block_table,
                const c10::optional<at::Tensor>& k_descale, const c10::optional<at::Tensor>& v_descale,
                const c10::optional<at::Tensor>& cu_seqlens_q, int64_t max_seqlen_q,
                const c10::optional<at::Tensor>& rotary_cos, const c10::optional<at::Tensor>& rotary_sin,
                const c10::optional<at::Tensor>& rotary_seqlens, bool rotary_interleaved,
                const c10::optional<at::Tensor>& q_descale, const c10::optional<at::Tensor>& cache_batch_idx,
                const c10::optional<at::Tensor>& cache_leftpad, const c10::optional<at::Tensor>& tree_mask) {
  const c10::cuda::CUDAGuard guard(q_in.device());
  const bool varlen = cu_seqlens_q.has_value();
  TORCH_CHECK(q_in.dim() == (varlen ? 3 : 4), "decode_fwd: q must be (B, Sq, Hq, D), or (total_q, Hq, D) with "
              "cu_seqlens_q");
  const int64_t total_q = varlen ? q_in.size(0) : 0;
  if (varlen) {
    const at::Tensor& cu = *cu_seqlens_q;
    TORCH_CHECK(cu.scalar_type() == at::kInt && cu.device() == q_in.device() && cu.is_contiguous() && cu.dim() == 1 &&
                    cu.numel() == seqlens.numel() + 1,
                "decode_fwd: cu_seqlens_q must be (B + 1,) int32 contiguous on q's device");
    TORCH_CHECK(max_seqlen_q >= 1, "decode_fwd: max_seqlen_q must be >= 1");
  }
  // the kernel's uniform view (B, Sq): varlen q as (1, total_q) for the shape checks below
  const at::Tensor q = varlen ? q_in.unsqueeze(0) : q_in;
  TORCH_CHECK(k_cache.dim() == 4 && v_cache.dim() == 4, "decode_fwd: 4-D k_cache / v_cache");
  TORCH_CHECK(k_cache.sizes() == v_cache.sizes(), "decode_fwd: k_cache and v_cache shapes differ");
  const bool fp8 = k_cache.scalar_type() == at::kFloat8_e4m3fn;
  const bool q8 = q.scalar_type() == at::kFloat8_e4m3fn;
  TORCH_CHECK(k_cache.scalar_type() == v_cache.scalar_type() && (fp8 || k_cache.scalar_type() == q.scalar_type()),
              "decode_fwd: caches must both have q's dtype or both be fp8 (float8_e4m3fn)");
  TORCH_CHECK(!q8 || fp8, "decode_fwd: an fp8 (float8_e4m3fn) q needs fp8 caches");
  TORCH_CHECK(k_descale.has_value() == fp8 && v_descale.has_value() == fp8,
              "decode_fwd: fp8 caches need k_descale and v_descale, and other caches take none");
  TORCH_CHECK(q_descale.has_value() == q8, "decode_fwd: an fp8 q needs q_descale, and other queries take none");
  const int64_t B = varlen ? seqlens.numel() : q.size(0);
  const int64_t sq = varlen ? max_seqlen_q : q.size(1), hq = q.size(2), d = q.size(3);
  const int64_t rows = varlen ? total_q : B * sq;  // packed query rows
  const bool paged = block_table.has_value();
  const int64_t page_size = paged ? k_cache.size(1) : 0;
  const int64_t s_cap = paged ? block_table->size(1) * page_size : k_cache.size(1);
  const int64_t hkv = k_cache.size(2);
  const int64_t cache_rows = k_cache.size(0) * k_cache.size(1);
  const bool slots = cache_batch_idx.has_value();
  TORCH_CHECK((paged || slots || k_cache.size(0) == B) && k_cache.size(3) == d,
              "decode_fwd: cache shape does not match q");
  TORCH_CHECK(!paged || (!slots && !cache_leftpad.has_value()),
              "decode_fwd: cache_batch_idx and cache_leftpad take a contiguous cache, not a block table");
  for (const c10::optional<at::Tensor>* t : {&cache_batch_idx, &cache_leftpad})
    TORCH_CHECK(!t->has_value() || ((*t)->scalar_type() == at::kInt && (*t)->device() == q.device() &&
                                    (*t)->dim() == 1 && (*t)->numel() == B && (*t)->is_contiguous()),
                "decode_fwd: cache_batch_idx / cache_leftpad must be (B,) int32 contiguous on q's device");
  // the TMA row coordinate of a contiguous cache is an int32
  TORCH_CHECK(paged || !slots || cache_rows < (int64_t(1) << 31),
              "decode_fwd: with cache_batch_idx, B_cache * S_cap must be below 2^31");
  TORCH_CHECK(q.stride(3) == 1 && (varlen || q.stride(0) == sq * q.stride(1)),
              "decode_fwd: q must be (B, Sq) mergeable");
  TORCH_CHECK((q.stride(1) * q.element_size()) % 16 == 0 && (q.stride(2) * q.element_size()) % 16 == 0 &&
                  reinterpret_cast<uintptr_t>(q.data_ptr()) % 16 == 0,
              "decode_fwd: q rows must be 16-byte aligned");
  for (const at::Tensor* c : {&k_cache, &v_cache})
    TORCH_CHECK(c->stride(3) == 1 && c->stride(0) == c->size(1) * c->stride(1),
                "decode_fwd: the cache's first two dimensions must be mergeable (stride(0) == size(1) * stride(1))");
  if (paged) {
    const at::Tensor& bt = *block_table;
    TORCH_CHECK(bt.scalar_type() == at::kInt && bt.is_cuda() && bt.device() == q.device() && bt.dim() == 2 &&
                    bt.size(0) == B && bt.size(1) >= 1 && bt.stride(1) == 1,
                "decode_fwd: block_table must be (B, max_blocks) int32 on q's device with stride(1) == 1");
    TORCH_CHECK(page_size == 16 || page_size == 32 || page_size == 64 || (page_size > 0 && page_size % 128 == 0),
                "decode_fwd: page_size must be 16, 32, 64 or a positive multiple of 128");
    TORCH_CHECK(cache_rows < (int64_t(1) << 31) && s_cap < (int64_t(1) << 31),
                "decode_fwd: num_blocks * page_size and max_blocks * page_size must be below 2^31");
  }
  TORCH_CHECK(seqlens.scalar_type() == at::kInt && seqlens.is_cuda() && seqlens.is_contiguous() && seqlens.numel() == B,
              "decode_fwd: cache_seqlens must be (B,) int32 on the device");
  // the kernel stores out as float2: every split's partial must start 8-byte aligned
  TORCH_CHECK(part.scalar_type() == at::kFloat && part.dim() == 2 && part.size(0) >= 1 && part.stride(1) == 1 &&
                  part.size(1) == rows * hq * d + rows * hq && part.stride(0) >= part.size(1) &&
                  part.stride(0) % 2 == 0 && reinterpret_cast<uintptr_t>(part.data_ptr()) % 8 == 0,
              "decode_fwd: part must be fp32 (n_splits, B*Sq*Hq*D + B*Hq*Sq), or total_q for B*Sq when varlen, with "
              "stride(1) == 1, an even stride(0) and an 8-byte aligned start");
  TORCH_CHECK(k_new.has_value() == v_new.has_value(), "decode_fwd: pass both k_new and v_new or neither");
  const void* kn = nullptr;
  const void* vn = nullptr;
  int new_dtype = q8 ? rfa::kDtypeE4M3 : dtype_code(q);
  if (k_new.has_value()) {
    // q's dtype; e4m3 over an e4m3 cache (stored as they are); bf16 / fp16 with an e4m3 q (quantised)
    const at::ScalarType nt = k_new->scalar_type();
    const bool nt_ok = nt == q.scalar_type() || (fp8 && nt == at::kFloat8_e4m3fn) ||
                       (q8 && (nt == at::kBFloat16 || nt == at::kHalf));
    for (const at::Tensor* t : {&*k_new, &*v_new}) {
      const bool shape_ok = varlen ? t->dim() == 3 && t->size(0) == total_q && t->size(1) == hkv && t->size(2) == d
                                   : t->dim() == 4 && t->size(0) == B && t->size(1) == sq && t->size(2) == hkv &&
                                         t->size(3) == d;
      TORCH_CHECK(t->is_contiguous() && t->scalar_type() == nt && nt_ok && shape_ok,
                  "decode_fwd: k_new / v_new must be contiguous (B, Sq, Hkv, D), or varlen (total_q, Hkv, D), in "
                  "q's dtype, or both e4m3 over e4m3 caches, or bf16 / fp16 with an e4m3 q");
    }
    new_dtype = nt == at::kFloat8_e4m3fn ? rfa::kDtypeE4M3 : dtype_code(*k_new);
    kn = k_new->data_ptr();
    vn = v_new->data_ptr();
  }
  const int64_t n_splits = part.size(0);
  const int64_t tiles = (s_cap + 127) / 128;
  rfa::DecodeParams p{};
  p.q = q.data_ptr();
  p.q_row_stride = q.stride(1);
  p.q_head_stride = q.stride(2);
  p.seqlens = seqlens.data_ptr<int>();
  p.part = part.data_ptr<float>();
  p.part_stride = part.stride(0);
  p.batch = static_cast<int>(B);
  p.sq = static_cast<int>(sq);
  p.hq = static_cast<int>(hq);
  p.hkv = static_cast<int>(hkv);
  p.cu_seqlens_q = varlen ? cu_seqlens_q->data_ptr<int>() : nullptr;
  p.total_q = static_cast<int>(rows);
  p.s_cap = static_cast<int>(s_cap);
  p.tiles_per_split = static_cast<int>((tiles + n_splits - 1) / n_splits);
  p.n_new = kn != nullptr ? static_cast<int>(sq) : 0;
  p.causal = causal ? 1 : 0;
  p.scale_log2 = static_cast<float>(scale * 1.4426950408889634);
  if (paged) {
    p.block_table = block_table->data_ptr<int>();
    p.bt_stride = block_table->stride(0);
    p.page_size = static_cast<int>(page_size);
    p.num_pages = static_cast<int>(k_cache.size(0));
  }
  if (fp8) {
    for (const at::Tensor* t : {&*k_descale, &*v_descale})
      TORCH_CHECK(t->scalar_type() == at::kFloat && t->is_cuda() && t->device() == q.device() && t->dim() == 2 &&
                      t->size(0) == B && t->size(1) == hkv && t->is_contiguous(),
                  "decode_fwd: fp8 descales must be contiguous fp32 (B, Hkv) on q's device");
    p.k_descale = k_descale->data_ptr<float>();
    p.v_descale = v_descale->data_ptr<float>();
  }
  if (q8) {
    const at::Tensor& t = *q_descale;
    TORCH_CHECK(t.scalar_type() == at::kFloat && t.is_cuda() && t.device() == q.device() && t.dim() == 2 &&
                    t.size(0) == B && t.size(1) == hkv && t.is_contiguous(),
                "decode_fwd: q_descale must be contiguous fp32 (B, Hkv) on q's device");
    p.q_descale = t.data_ptr<float>();
  }
  TORCH_CHECK(rotary_cos.has_value() == rotary_sin.has_value() && rotary_cos.has_value() == rotary_seqlens.has_value(),
              "decode_fwd: rotary needs rotary_cos, rotary_sin and rotary_seqlens together");
  if (rotary_cos.has_value()) {
    TORCH_CHECK(!q8 && new_dtype != rfa::kDtypeE4M3,
                "decode_fwd: rotary needs a bf16 / fp16 q and k_new (rotate before quantising)");
    const at::Tensor& rc = *rotary_cos;
    const at::Tensor& rs = *rotary_sin;
    TORCH_CHECK(rc.dim() == 2 && rc.sizes() == rs.sizes() && rc.size(0) >= 1 && rc.is_contiguous() &&
                    rs.is_contiguous() && rc.scalar_type() == q.scalar_type() &&
                    rs.scalar_type() == q.scalar_type() && rc.device() == q.device() && rs.device() == q.device(),
                "decode_fwd: rotary_cos / rotary_sin must be contiguous (seqlen_ro, rotary_dim / 2) in q's dtype on "
                "q's device");
    TORCH_CHECK(rc.size(1) >= 8 && rc.size(1) % 8 == 0 && 2 * rc.size(1) <= d,
                "decode_fwd: rotary_dim must be a positive multiple of 16, at most head_dim");
    TORCH_CHECK(rc.size(0) < (int64_t(1) << 31), "decode_fwd: seqlen_ro must be below 2^31");
    const at::Tensor& rsl = *rotary_seqlens;
    TORCH_CHECK(rsl.scalar_type() == at::kInt && rsl.device() == q.device() && rsl.is_contiguous() && rsl.dim() == 1 &&
                    rsl.numel() == B,
                "decode_fwd: rotary_seqlens must be (B,) int32 contiguous on q's device");
    p.rotary_cos = rc.data_ptr();
    p.rotary_sin = rs.data_ptr();
    p.rotary_seqlens = rsl.data_ptr<int>();
    p.rotary_half = static_cast<int>(rc.size(1));
    p.seqlen_ro = static_cast<int>(rc.size(0));
    p.rotary_interleaved = rotary_interleaved ? 1 : 0;
  }
  if (slots) {
    p.cache_batch_idx = cache_batch_idx->data_ptr<int>();
    p.cache_batch = static_cast<int>(k_cache.size(0));
  }
  if (cache_leftpad.has_value()) p.cache_leftpad = cache_leftpad->data_ptr<int>();
  p.tree_mask = tree_mask_ptr(tree_mask, q, rows, sq, causal, "decode_fwd");
  const TensorView kv{k_cache.data_ptr(), cache_rows, static_cast<int>(hkv), k_cache.stride(1), k_cache.stride(2)};
  const TensorView vv{v_cache.data_ptr(), cache_rows, static_cast<int>(hkv), v_cache.stride(1), v_cache.stride(2)};
  check(rfa::decode_fwd_launch(q8 ? rfa::kDtypeE4M3 : dtype_code(q), fp8 ? rfa::kDtypeE4M3 : dtype_code(q), kv, vv,
                               kn, vn, new_dtype, p, static_cast<int>(n_splits), static_cast<int>(d),
                               at::cuda::getCurrentCUDAStream()));
}

// The shared-prefix pass of split-KV decode (see decode_prefix_launch): attention of q (B, Sq, Hq, D), or varlen
// (total_q, Hq, D) with cu_seqlens_q (B + 1,), to P shared prefixes prefix_k / prefix_v (P, P_cap, Hkv, D) with
// mergeable first two dimensions, in q's dtype or both e4m3 with k_descale / v_descale fp32 (P, Hkv) contiguous.
// Sequence b reads prefix b / (B / P), rows [0, prefix_seqlens[p]) (read on the device only, clamped to [0, P_cap]),
// all visible to every query token.  part: the partial slabs of this pass, in decode_fwd's layout.  causal and the
// rotary tensors position q's rotation as in decode_fwd, and so does tree_mask (which masks no prefix key).  With
// prefix_block_table (P, max_prefix_blocks) int32, prefix_k / prefix_v are page pools (num_blocks, page_size, Hkv, D)
// with mergeable page and row dimensions (they may be decode_fwd's own pools), row j of prefix p lives at row
// j % page_size of page prefix_block_table[p, j / page_size], and P_cap = max_prefix_blocks * page_size.
void decode_prefix_fwd(const at::Tensor& q_in, const at::Tensor& prefix_k, const at::Tensor& prefix_v,
                       const at::Tensor& prefix_seqlens, bool causal, double scale, at::Tensor& part,
                       const c10::optional<at::Tensor>& k_descale, const c10::optional<at::Tensor>& v_descale,
                       const c10::optional<at::Tensor>& cu_seqlens_q, int64_t max_seqlen_q,
                       const c10::optional<at::Tensor>& rotary_cos, const c10::optional<at::Tensor>& rotary_sin,
                       const c10::optional<at::Tensor>& rotary_seqlens, bool rotary_interleaved,
                       const c10::optional<at::Tensor>& tree_mask,
                       const c10::optional<at::Tensor>& prefix_block_table) {
  const c10::cuda::CUDAGuard guard(q_in.device());
  const bool varlen = cu_seqlens_q.has_value();
  TORCH_CHECK(q_in.dim() == (varlen ? 3 : 4), "decode_prefix_fwd: q must be (B, Sq, Hq, D), or (total_q, Hq, D) "
              "with cu_seqlens_q");
  TORCH_CHECK(q_in.scalar_type() == at::kBFloat16 || q_in.scalar_type() == at::kHalf,
              "decode_prefix_fwd: q must be bf16 or fp16");
  const int64_t total_q = varlen ? q_in.size(0) : 0;
  if (varlen) {
    const at::Tensor& cu = *cu_seqlens_q;
    TORCH_CHECK(cu.scalar_type() == at::kInt && cu.device() == q_in.device() && cu.is_contiguous() && cu.dim() == 1 &&
                    cu.numel() >= 2,
                "decode_prefix_fwd: cu_seqlens_q must be (B + 1,) int32 contiguous on q's device");
    TORCH_CHECK(max_seqlen_q >= 1, "decode_prefix_fwd: max_seqlen_q must be >= 1");
  }
  const at::Tensor q = varlen ? q_in.unsqueeze(0) : q_in;
  const int64_t B = varlen ? cu_seqlens_q->numel() - 1 : q.size(0);
  const int64_t sq = varlen ? max_seqlen_q : q.size(1), hq = q.size(2), d = q.size(3);
  const int64_t rows = varlen ? total_q : B * sq;
  TORCH_CHECK(prefix_k.dim() == 4 && prefix_k.sizes() == prefix_v.sizes(),
              "decode_prefix_fwd: prefix_k / prefix_v must be the same (P, P_cap, Hkv, D) shape, or the same "
              "(num_blocks, page_size, Hkv, D) shape with prefix_block_table");
  const bool paged = prefix_block_table.has_value();
  const int64_t page_size = paged ? prefix_k.size(1) : 0;
  const int64_t n_prefix = paged ? prefix_block_table->size(0) : prefix_k.size(0);
  const int64_t p_cap = paged ? prefix_block_table->size(1) * page_size : prefix_k.size(1);
  const int64_t hkv = prefix_k.size(2);
  const int64_t cache_rows = prefix_k.size(0) * prefix_k.size(1);  // a contiguous cache's P * P_cap
  if (paged) {
    const at::Tensor& bt = *prefix_block_table;
    TORCH_CHECK(bt.scalar_type() == at::kInt && bt.is_cuda() && bt.device() == q_in.device() && bt.dim() == 2 &&
                    bt.size(0) >= 1 && bt.size(1) >= 1 && bt.stride(1) == 1,
                "decode_prefix_fwd: prefix_block_table must be (P, max_prefix_blocks) int32 on q's device with "
                "stride(1) == 1");
    TORCH_CHECK(page_size == 16 || page_size == 32 || page_size == 64 || (page_size > 0 && page_size % 128 == 0),
                "decode_prefix_fwd: page_size must be 16, 32, 64 or a positive multiple of 128");
    TORCH_CHECK(cache_rows < (int64_t(1) << 31) && p_cap < (int64_t(1) << 31),
                "decode_prefix_fwd: num_blocks * page_size and max_prefix_blocks * page_size must be below 2^31");
  }
  const bool fp8 = prefix_k.scalar_type() == at::kFloat8_e4m3fn;
  TORCH_CHECK(prefix_k.scalar_type() == prefix_v.scalar_type() && (fp8 || prefix_k.scalar_type() == q.scalar_type()),
              "decode_prefix_fwd: the prefix caches must both have q's dtype or both be fp8 (float8_e4m3fn)");
  TORCH_CHECK(k_descale.has_value() == fp8 && v_descale.has_value() == fp8,
              "decode_prefix_fwd: fp8 prefix caches need k_descale and v_descale, and other caches take none");
  TORCH_CHECK(n_prefix >= 1 && B % n_prefix == 0 && prefix_k.size(3) == d && hkv >= 1 && hq % hkv == 0,
              "decode_prefix_fwd: the prefix caches do not match q (P must divide B)");
  TORCH_CHECK(paged || cache_rows < (int64_t(1) << 31), "decode_prefix_fwd: P * P_cap must be below 2^31");
  TORCH_CHECK(q.stride(3) == 1 && (varlen || q.stride(0) == sq * q.stride(1)),
              "decode_prefix_fwd: q must be (B, Sq) mergeable");
  TORCH_CHECK((q.stride(1) * q.element_size()) % 16 == 0 && (q.stride(2) * q.element_size()) % 16 == 0 &&
                  reinterpret_cast<uintptr_t>(q.data_ptr()) % 16 == 0,
              "decode_prefix_fwd: q rows must be 16-byte aligned");
  for (const at::Tensor* c : {&prefix_k, &prefix_v})
    TORCH_CHECK(c->device() == q.device() && c->stride(3) == 1 && c->stride(0) == c->size(1) * c->stride(1),
                "decode_prefix_fwd: the prefix caches must be on q's device with mergeable first two dimensions");
  TORCH_CHECK(prefix_seqlens.scalar_type() == at::kInt && prefix_seqlens.device() == q.device() &&
                  prefix_seqlens.is_contiguous() && prefix_seqlens.dim() == 1 && prefix_seqlens.numel() == n_prefix,
              "decode_prefix_fwd: prefix_seqlens must be (P,) int32 contiguous on q's device");
  TORCH_CHECK(part.scalar_type() == at::kFloat && part.dim() == 2 && part.size(0) >= 1 && part.stride(1) == 1 &&
                  part.size(1) == rows * hq * d + rows * hq && part.stride(0) >= part.size(1) &&
                  part.stride(0) % 2 == 0 && reinterpret_cast<uintptr_t>(part.data_ptr()) % 8 == 0,
              "decode_prefix_fwd: part must be fp32 (n_splits, B*Sq*Hq*D + B*Hq*Sq), or total_q for B*Sq when "
              "varlen, with stride(1) == 1, an even stride(0) and an 8-byte aligned start");
  const int64_t n_splits = part.size(0);
  const int64_t tiles = (p_cap + 127) / 128;
  rfa::DecodeParams p{};
  p.q = q.data_ptr();
  p.q_row_stride = q.stride(1);
  p.q_head_stride = q.stride(2);
  p.seqlens = prefix_seqlens.data_ptr<int>();
  p.part = part.data_ptr<float>();
  p.part_stride = part.stride(0);
  p.batch = static_cast<int>(B);
  p.sq = static_cast<int>(sq);
  p.hq = static_cast<int>(hq);
  p.hkv = static_cast<int>(hkv);
  p.cu_seqlens_q = varlen ? cu_seqlens_q->data_ptr<int>() : nullptr;
  p.total_q = static_cast<int>(rows);
  p.s_cap = static_cast<int>(p_cap);
  p.tiles_per_split = static_cast<int>(std::max<int64_t>(1, (tiles + n_splits - 1) / n_splits));
  p.n_new = 0;
  p.causal = causal ? 1 : 0;
  p.scale_log2 = static_cast<float>(scale * 1.4426950408889634);
  p.prefix_n = static_cast<int>(B / n_prefix);
  if (paged) {
    p.block_table = prefix_block_table->data_ptr<int>();
    p.bt_stride = prefix_block_table->stride(0);
    p.page_size = static_cast<int>(page_size);
    p.num_pages = static_cast<int>(prefix_k.size(0));
  }
  if (fp8) {
    for (const at::Tensor* t : {&*k_descale, &*v_descale})
      TORCH_CHECK(t->scalar_type() == at::kFloat && t->device() == q.device() && t->dim() == 2 &&
                      t->size(0) == n_prefix && t->size(1) == hkv && t->is_contiguous(),
                  "decode_prefix_fwd: fp8 descales must be contiguous fp32 (P, Hkv) on q's device");
    p.k_descale = k_descale->data_ptr<float>();
    p.v_descale = v_descale->data_ptr<float>();
  }
  TORCH_CHECK(rotary_cos.has_value() == rotary_sin.has_value() && rotary_cos.has_value() == rotary_seqlens.has_value(),
              "decode_prefix_fwd: rotary needs rotary_cos, rotary_sin and rotary_seqlens together");
  if (rotary_cos.has_value()) {
    const at::Tensor& rc = *rotary_cos;
    const at::Tensor& rs = *rotary_sin;
    TORCH_CHECK(rc.dim() == 2 && rc.sizes() == rs.sizes() && rc.size(0) >= 1 && rc.is_contiguous() &&
                    rs.is_contiguous() && rc.scalar_type() == q.scalar_type() &&
                    rs.scalar_type() == q.scalar_type() && rc.device() == q.device() && rs.device() == q.device(),
                "decode_prefix_fwd: rotary_cos / rotary_sin must be contiguous (seqlen_ro, rotary_dim / 2) in q's "
                "dtype on q's device");
    TORCH_CHECK(rc.size(1) >= 8 && rc.size(1) % 8 == 0 && 2 * rc.size(1) <= d,
                "decode_prefix_fwd: rotary_dim must be a positive multiple of 16, at most head_dim");
    TORCH_CHECK(rc.size(0) < (int64_t(1) << 31), "decode_prefix_fwd: seqlen_ro must be below 2^31");
    const at::Tensor& rsl = *rotary_seqlens;
    TORCH_CHECK(rsl.scalar_type() == at::kInt && rsl.device() == q.device() && rsl.is_contiguous() && rsl.dim() == 1 &&
                    rsl.numel() == B,
                "decode_prefix_fwd: rotary_seqlens must be (B,) int32 contiguous on q's device");
    p.rotary_cos = rc.data_ptr();
    p.rotary_sin = rs.data_ptr();
    p.rotary_seqlens = rsl.data_ptr<int>();
    p.rotary_half = static_cast<int>(rc.size(1));
    p.seqlen_ro = static_cast<int>(rc.size(0));
    p.rotary_interleaved = rotary_interleaved ? 1 : 0;
  }
  p.tree_mask = tree_mask_ptr(tree_mask, q, rows, sq, causal, "decode_prefix_fwd");
  const TensorView kv{prefix_k.data_ptr(), cache_rows, static_cast<int>(hkv), prefix_k.stride(1), prefix_k.stride(2)};
  const TensorView vv{prefix_v.data_ptr(), cache_rows, static_cast<int>(hkv), prefix_v.stride(1), prefix_v.stride(2)};
  check(rfa::decode_prefix_launch(dtype_code(q), fp8 ? rfa::kDtypeE4M3 : dtype_code(q), kv, vv, p,
                                  static_cast<int>(n_prefix), static_cast<int>(n_splits), static_cast<int>(d),
                                  at::cuda::getCurrentCUDAStream()));
}

// Merges the partials of decode_fwd (or gathered per-rank partials, same layout): out (B, Sq, Hq, D) contiguous in
// bf16 / fp16 / fp32, lse (B, Hq, Sq) fp32 contiguous.
void decode_combine(const at::Tensor& parts, at::Tensor& out, at::Tensor& lse) {
  const c10::cuda::CUDAGuard guard(parts.device());
  TORCH_CHECK(out.dim() == 4 && out.is_contiguous() && out.is_cuda(), "decode_combine: out must be contiguous (B, Sq, Hq, D)");
  const int64_t B = out.size(0), sq = out.size(1), hq = out.size(2), d = out.size(3);
  TORCH_CHECK(parts.scalar_type() == at::kFloat && parts.dim() == 2 && parts.size(0) >= 1 && parts.stride(1) == 1 &&
                  parts.stride(0) >= parts.size(1) && parts.size(1) == B * sq * hq * d + B * hq * sq,
              "decode_combine: parts must be fp32 (P, B*Sq*Hq*D + B*Hq*Sq) with stride(1) == 1");
  TORCH_CHECK(lse.scalar_type() == at::kFloat && lse.is_contiguous() && lse.numel() == B * hq * sq,
              "decode_combine: lse must be fp32 (B, Hq, Sq)");
  const int out_dtype = out.scalar_type() == at::kFloat ? -1 : dtype_code(out);
  check(rfa::decode_combine_launch(parts.data_ptr<float>(), parts.stride(0), static_cast<int>(parts.size(0)),
                                   static_cast<int>(B), static_cast<int>(sq), static_cast<int>(hq), static_cast<int>(d),
                                   out.data_ptr(), out_dtype, lse.data_ptr<float>(), at::cuda::getCurrentCUDAStream()));
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "ring_flash_attn_b200 sm_90a kernels";
  pybind11::class_<FusedCtx>(m, "FusedCtx")
      .def(pybind11::init<>())
      .def_readwrite("k_stage", &FusedCtx::k_stage)
      .def_readwrite("v_stage", &FusedCtx::v_stage)
      .def_readwrite("my_pad", &FusedCtx::my_pad)
      .def_readwrite("push_tasks", &FusedCtx::push_tasks)
      .def_readwrite("dyn_needs", &FusedCtx::dyn_needs)
      .def_readwrite("dyn_chunk_rows", &FusedCtx::dyn_chunk_rows)
      .def_readwrite("dyn_chunks", &FusedCtx::dyn_chunks)
      .def_readwrite("rows_cap", &FusedCtx::rows_cap)
      .def_readwrite("region_bytes", &FusedCtx::region_bytes)
      .def_readwrite("counters", &FusedCtx::counters)
      .def_readwrite("stage_ptrs", &FusedCtx::stage_ptrs)
      .def_readwrite("pad_ptrs", &FusedCtx::pad_ptrs)
      .def_readwrite("sent_targets", &FusedCtx::sent_targets)
      .def_readwrite("n_push_ctas", &FusedCtx::n_push_ctas)
      .def_readwrite("row_bytes", &FusedCtx::row_bytes)
      .def_readwrite("my_rank", &FusedCtx::my_rank)
      .def_readwrite("world", &FusedCtx::world)
      .def_readwrite("epoch", &FusedCtx::epoch)
      .def_readwrite("done_target", &FusedCtx::done_target)
      .def_readwrite("parity_off", &FusedCtx::parity_off)
      .def_readwrite("dk_ptrs", &FusedCtx::dk_ptrs)
      .def_readwrite("dv_ptrs", &FusedCtx::dv_ptrs)
      .def_readwrite("dkv_targets", &FusedCtx::dkv_targets)
      .def_readwrite("dkv_wait_epoch", &FusedCtx::dkv_wait_epoch);
  m.attr("NEED_RANGES") = rfa::kNeedRanges;
  m.def("set_trace", &set_trace);
  m.def("attn_fwd", &attn_fwd);
  m.def("attn_fwd_window", &attn_fwd_window);
  m.def("attn_fwd_fp8", &attn_fwd_fp8);
  m.def("attn_fwd_fused_fp8", &attn_fwd_fused_fp8);
  m.def("attn_bwd_window", &attn_bwd_window);
  m.def("attn_fwd_fused", &attn_fwd_fused);
  m.def("attn_fwd_fused_window", &attn_fwd_fused_window);
  m.def("attn_bwd_fused_window", &attn_bwd_fused_window);
  m.def("attn_bwd_fused", &attn_bwd_fused);
  m.def("reduce_dkv", &reduce_dkv);
  m.def("dq_finalize", &dq_finalize);
  m.def("attn_bwd_delta", &attn_bwd_delta);
  m.def("attn_bwd", &attn_bwd);
  m.def("lse_flatten", &lse_flatten);
  m.def("lse_unflatten", &lse_unflatten);
  m.def("decode_fwd", &decode_fwd);
  // the same without tree_mask
  m.def("decode_fwd", [](const at::Tensor& q, at::Tensor& k_cache, at::Tensor& v_cache, const at::Tensor& seqlens,
                         const c10::optional<at::Tensor>& k_new, const c10::optional<at::Tensor>& v_new, bool causal,
                         double scale, at::Tensor& part, const c10::optional<at::Tensor>& block_table,
                         const c10::optional<at::Tensor>& k_descale, const c10::optional<at::Tensor>& v_descale,
                         const c10::optional<at::Tensor>& cu_seqlens_q, int64_t max_seqlen_q,
                         const c10::optional<at::Tensor>& rotary_cos, const c10::optional<at::Tensor>& rotary_sin,
                         const c10::optional<at::Tensor>& rotary_seqlens, bool rotary_interleaved,
                         const c10::optional<at::Tensor>& q_descale, const c10::optional<at::Tensor>& cache_batch_idx,
                         const c10::optional<at::Tensor>& cache_leftpad) {
    decode_fwd(q, k_cache, v_cache, seqlens, k_new, v_new, causal, scale, part, block_table, k_descale, v_descale,
               cu_seqlens_q, max_seqlen_q, rotary_cos, rotary_sin, rotary_seqlens, rotary_interleaved, q_descale,
               cache_batch_idx, cache_leftpad, c10::nullopt);
  });
  // the same without cache_batch_idx / cache_leftpad
  m.def("decode_fwd", [](const at::Tensor& q, at::Tensor& k_cache, at::Tensor& v_cache, const at::Tensor& seqlens,
                         const c10::optional<at::Tensor>& k_new, const c10::optional<at::Tensor>& v_new, bool causal,
                         double scale, at::Tensor& part, const c10::optional<at::Tensor>& block_table,
                         const c10::optional<at::Tensor>& k_descale, const c10::optional<at::Tensor>& v_descale,
                         const c10::optional<at::Tensor>& cu_seqlens_q, int64_t max_seqlen_q,
                         const c10::optional<at::Tensor>& rotary_cos, const c10::optional<at::Tensor>& rotary_sin,
                         const c10::optional<at::Tensor>& rotary_seqlens, bool rotary_interleaved,
                         const c10::optional<at::Tensor>& q_descale) {
    decode_fwd(q, k_cache, v_cache, seqlens, k_new, v_new, causal, scale, part, block_table, k_descale, v_descale,
               cu_seqlens_q, max_seqlen_q, rotary_cos, rotary_sin, rotary_seqlens, rotary_interleaved, q_descale,
               c10::nullopt, c10::nullopt, c10::nullopt);
  });
  // the same without q_descale (a bf16 / fp16 q)
  m.def("decode_fwd", [](const at::Tensor& q, at::Tensor& k_cache, at::Tensor& v_cache, const at::Tensor& seqlens,
                         const c10::optional<at::Tensor>& k_new, const c10::optional<at::Tensor>& v_new, bool causal,
                         double scale, at::Tensor& part, const c10::optional<at::Tensor>& block_table,
                         const c10::optional<at::Tensor>& k_descale, const c10::optional<at::Tensor>& v_descale,
                         const c10::optional<at::Tensor>& cu_seqlens_q, int64_t max_seqlen_q,
                         const c10::optional<at::Tensor>& rotary_cos, const c10::optional<at::Tensor>& rotary_sin,
                         const c10::optional<at::Tensor>& rotary_seqlens, bool rotary_interleaved) {
    decode_fwd(q, k_cache, v_cache, seqlens, k_new, v_new, causal, scale, part, block_table, k_descale, v_descale,
               cu_seqlens_q, max_seqlen_q, rotary_cos, rotary_sin, rotary_seqlens, rotary_interleaved, c10::nullopt,
               c10::nullopt, c10::nullopt, c10::nullopt);
  });
  m.def("decode_prefix_fwd", &decode_prefix_fwd);
  // the same without prefix_block_table (a contiguous prefix)
  m.def("decode_prefix_fwd", [](const at::Tensor& q, const at::Tensor& prefix_k, const at::Tensor& prefix_v,
                                const at::Tensor& prefix_seqlens, bool causal, double scale, at::Tensor& part,
                                const c10::optional<at::Tensor>& k_descale, const c10::optional<at::Tensor>& v_descale,
                                const c10::optional<at::Tensor>& cu_seqlens_q, int64_t max_seqlen_q,
                                const c10::optional<at::Tensor>& rotary_cos,
                                const c10::optional<at::Tensor>& rotary_sin,
                                const c10::optional<at::Tensor>& rotary_seqlens, bool rotary_interleaved,
                                const c10::optional<at::Tensor>& tree_mask) {
    decode_prefix_fwd(q, prefix_k, prefix_v, prefix_seqlens, causal, scale, part, k_descale, v_descale, cu_seqlens_q,
                      max_seqlen_q, rotary_cos, rotary_sin, rotary_seqlens, rotary_interleaved, tree_mask,
                      c10::nullopt);
  });
  // the same without tree_mask
  m.def("decode_prefix_fwd", [](const at::Tensor& q, const at::Tensor& prefix_k, const at::Tensor& prefix_v,
                                const at::Tensor& prefix_seqlens, bool causal, double scale, at::Tensor& part,
                                const c10::optional<at::Tensor>& k_descale, const c10::optional<at::Tensor>& v_descale,
                                const c10::optional<at::Tensor>& cu_seqlens_q, int64_t max_seqlen_q,
                                const c10::optional<at::Tensor>& rotary_cos,
                                const c10::optional<at::Tensor>& rotary_sin,
                                const c10::optional<at::Tensor>& rotary_seqlens, bool rotary_interleaved) {
    decode_prefix_fwd(q, prefix_k, prefix_v, prefix_seqlens, causal, scale, part, k_descale, v_descale, cu_seqlens_q,
                      max_seqlen_q, rotary_cos, rotary_sin, rotary_seqlens, rotary_interleaved, c10::nullopt,
                      c10::nullopt);
  });
  m.def("decode_combine", &decode_combine);
  rfa::bind_peer_mem(m);
}
