// Python bindings for the sm_90a kernels and the peer-memory runtime (module ring_flash_attn_b200._C).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <cstdlib>

#include "attn_common.h"
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
  rfa::bind_peer_mem(m);
}
