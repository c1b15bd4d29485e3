"""fp8 (e4m3) queries over e4m3 caches (``q_descale``): the quantised query, a stand-in extension that takes it, and
the oracle run built on ``tests/decode_oracle.py``.

An e4m3 query stands for ``q.float() * q_descale[b, kv head]``.  :func:`quantise_q` quantises a case's bf16 query with
per-(sequence, kv head) descales that are not powers of two, and returns that fp64 dequantised query too: the
references of ``decode_oracle`` then run on it unchanged (fp64 scores, and fp32 scores of the dequantised query, P
rounded to bf16, bf16 V).  The kernel forms ``Q K^T`` as an e4m3 wgmma, which does not accumulate in full fp32, so
the bound is ``kernel_oracle``'s e4m3 allowance (``FP8_RATIO``, ``FP8_LSE_REL``).
"""
from __future__ import annotations

import dataclasses

import torch

import decode_oracle as DO
import kernel_oracle as KO
from fake_ext import FakeDecodeExt
from ring_flash_attn_b200.parallel import decode as dec
from test_gpu_decode_fp8 import bytes_of

E4M3 = torch.float8_e4m3fn


def quantise_q(inp: DO.Inputs):
    """(q8 (rows, Hq, D) e4m3, q_descale (B, Hkv) fp32, the dequantised q in fp64) for a case's query: each
    (sequence, kv head) scaled so that its largest element lands between 400 and 448."""
    case, d = inp.case, inp.d
    g, hkv = case.group, case.hkv
    qf = inp.q.float()
    qd = torch.ones(case.b, hkv, dtype=torch.float32, device=qf.device)
    for i, (lo, n) in enumerate(DO.spans(case)):
        if n:
            amax = qf[lo:lo + n].view(n, hkv, g, d).abs().amax(dim=(0, 2, 3)).clamp(min=1e-3)
            qd[i] = amax / 448 * (1 + 0.1 * torch.arange(hkv, device=qf.device) / hkv)
    per_head = qd.repeat_interleave(g, dim=1)  # (B, Hq)
    q8 = torch.cat([(qf[lo:lo + n] / per_head[i][:, None]).clamp(-448, 448).to(E4M3)
                    for i, (lo, n) in enumerate(DO.spans(case))])
    q64 = torch.cat([q8[lo:lo + n].double() * per_head[i].double()[:, None]
                     for i, (lo, n) in enumerate(DO.spans(case))])
    return q8, qd, q64


def run_q8(case: DO.Case, d: int, regime: str, device, append_kind: str = "bf16", seed: int = 0):
    """One e4m3-query case through ``kernel_decode`` against both references, then the cache bytes.  ``append_kind``:
    "bf16" (quantised by the append) or "e4m3" (stored as they are)."""
    case = dataclasses.replace(case, fp8=True)
    assert case.rotary is None
    inp = DO.build_inputs(case, torch.bfloat16, d, regime, device, seed)
    q8, qd, q64 = quantise_q(inp)
    n_splits = case.splits if case.splits is not None else DO.default_splits(case, device)
    k0, v0 = inp.k_cache.clone(), inp.v_cache.clone()
    src = dataclasses.replace(inp, q=q8)
    if case.append and append_kind == "e4m3":
        src = dataclasses.replace(src, k_new=inp.stored_k, v_new=inp.stored_v)
    q, k, v = DO.call_views(src, case.append)
    splits = case.splits if torch.device(device).type == "cuda" else n_splits
    out, lse = dec.kernel_decode(q, inp.k_cache, inp.v_cache, inp.seqlens, k, v, case.causal, d ** -0.5,
                                 splits=splits, q_descale=qd, **DO.call_kwargs(inp))
    o64, l64, o32, l32 = DO.references(dataclasses.replace(inp, q=q64), n_splits)
    tag = f"decode q8 {case.name} D{d} {regime} append {append_kind}"
    assert out.dtype == torch.bfloat16 and out.shape == q.shape, (tag, out.dtype, out.shape)
    got_o, got_l = DO.packed(case, out, lse)
    KO.assert_accurate(f"{tag}: out", got_o, o64, o32.to(torch.bfloat16),
                       factor=max(KO.FP8_RATIO, KO._factor(regime)),
                       report=f"decode e4m3-q D{d}" + (" (large)" if regime == "large" else ""))
    KO.assert_lse(f"{tag}: lse", got_l, l64, l32, rel_limit=KO.FP8_LSE_REL, report="decode lse e4m3-q")
    want_k, want_v = DO.expected_caches(inp, k0, v0, case.append)
    for name, got, want in (("k_cache", inp.k_cache, want_k), ("v_cache", inp.v_cache, want_v)):
        diff = bytes_of(got) != bytes_of(want)
        assert not diff.any(), f"{tag}: {name} bytes differ at {diff.nonzero()[:4].tolist()}"


def run_two_ranks_q8(rank: int, world: int, device_type: str):
    """``decode_oracle.run_two_ranks`` with an e4m3 query (the same on both ranks) and e4m3 k / v appended on rank 1."""
    import torch.distributed as dist

    if device_type == "cpu":
        from ring_flash_attn_b200.ops import cuda_ext

        cuda_ext.load = FakeQ8DecodeExt
    else:
        torch.backends.cuda.matmul.allow_tf32 = False
    case = dataclasses.replace(DO.TWO_RANK_CASE, fp8=True)
    d, append_rank = 128, 1
    dev = f"cuda:{rank}" if device_type == "cuda" else "cpu"
    shards = [DO.build_inputs(case, torch.bfloat16, d, "randn", dev, seed=3, cache_seed=10 + r) for r in range(world)]
    inp = shards[rank]
    q8, qd, _ = quantise_q(inp)
    src = dataclasses.replace(inp, q=q8, k_new=inp.stored_k, v_new=inp.stored_v)
    q, k, v = DO.call_views(src, rank == append_rank)
    out, lse = dec.kernel_decode(q, inp.k_cache, inp.v_cache, inp.seqlens, k, v, case.causal, d ** -0.5,
                                 pg=dist.group.WORLD, world=world, splits=case.splits, q_descale=qd,
                                 **DO.call_kwargs(inp))
    refs = []
    for r, s in enumerate(shards):
        refs.append(DO.references(dataclasses.replace(s, q=quantise_q(s)[2]), case.splits,
                                  appended_here=r == append_rank))
    o64, l64 = DO.combine_ranks64([(a, b) for a, b, _, _ in refs])
    o32, l32 = DO.combine_ranks32([(c, e) for _, _, c, e in refs])
    got_o, got_l = DO.packed(case, out, lse)
    KO.assert_accurate("decode q8 two ranks: out", got_o, o64, o32.to(torch.bfloat16), factor=KO.FP8_RATIO)
    KO.assert_lse("decode q8 two ranks: lse", got_l, l64, l32, rel_limit=KO.FP8_LSE_REL)
    both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
    got = [torch.empty_like(both) for _ in range(world)]
    dist.all_gather(got, both)
    for x in got:
        assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0)), "the ranks' results differ"


class FakeQ8DecodeExt(FakeDecodeExt):
    """:class:`fake_ext.FakeDecodeExt` with the e4m3-query contract: ``q_descale`` multiplies the scores with
    ``k_descale``, P V runs in bf16, and e4m3 ``k_new`` / ``v_new`` are stored as they are."""

    def decode_fwd(self, q, k_cache, v_cache, seqlens, k_new, v_new, causal, scale, part, block_table, k_descale,
                   v_descale, cu_seqlens_q, max_seqlen_q, rotary_cos, rotary_sin, rotary_seqlens, rotary_interleaved,
                   q_descale=None):
        assert (q.dtype == E4M3) == (q_descale is not None)
        self._q_descale = q_descale
        self._pv_dtype = torch.bfloat16 if q.dtype == E4M3 else None
        self._appended = k_new is not None
        if k_new is not None and k_new.dtype == E4M3:
            assert rotary_cos is None and k_cache.dtype == E4M3
            self._copy_append(q, k_cache, v_cache, seqlens, k_new, v_new, block_table, cu_seqlens_q, max_seqlen_q)
            k_new = v_new = None  # the keys are in the cache; _n_vis still counts them
        super().decode_fwd(q, k_cache, v_cache, seqlens, k_new, v_new, causal, scale, part, block_table, k_descale,
                           v_descale, cu_seqlens_q, max_seqlen_q, rotary_cos, rotary_sin, rotary_seqlens,
                           rotary_interleaved)

    def _copy_append(self, q, k_cache, v_cache, seqlens, k_new, v_new, block_table, cu_seqlens_q, max_seqlen_q):
        nb = seqlens.numel()
        if cu_seqlens_q is not None:
            rows = q.shape[0]
            cu = [min(max(x, 0), rows) for x in cu_seqlens_q.tolist()]
            spans = [(cu[i], min(max(cu[i + 1] - cu[i], 0), max_seqlen_q)) for i in range(nb)]
        else:
            sq = q.shape[1]
            spans = [(i * sq, sq) for i in range(nb)]
            k_new, v_new = k_new.reshape(nb * sq, *k_new.shape[2:]), v_new.reshape(nb * sq, *v_new.shape[2:])
        paged = block_table is not None
        ps = k_cache.shape[1] if paged else 0
        s_cap = block_table.shape[1] * ps if paged else k_cache.shape[1]
        table = block_table.tolist() if paged else None
        for b, (lo, cnt) in enumerate(spans):
            for t in range(cnt):
                row = int(seqlens[b]) + t
                if not 0 <= row < s_cap:
                    continue
                at = (b, row)
                if paged:
                    page = table[b][row // ps]
                    if not 0 <= page < k_cache.shape[0]:
                        continue
                    at = (page, row % ps)
                k_cache[at] = k_new[lo + t]
                v_cache[at] = v_new[lo + t]

    def _n_vis(self, t, n_q, causal, appended):
        return super()._n_vis(t, n_q, causal, self._appended)

    def _k_descale(self, ds, b, kv_head):
        kd = ds[b, kv_head]
        return kd if self._q_descale is None else kd * self._q_descale[b, kv_head]

    def _p_for_pv(self, p, dtype):
        return super()._p_for_pv(p, self._pv_dtype or dtype)
