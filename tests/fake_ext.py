"""A torch implementation of the extension's launch entry points, driven by the SAME device work tables.

It lets the CPU suite run the code paths that normally need an H100 - table construction, launch dispatch
(plain / sliding-window / fp8), per-source ring steps, the autograd bridge - end to end against the dense oracle.
Each function implements the *contract* of its kernel (what the tables mean), not the tile schedule; the tile-level
index arithmetic is replayed separately in tests/test_tables.py.
"""
import torch

DIAG_FULL = 1 << 29
LO_NONE = -(1 << 29)


def _visible(n_rows, q_off, kv_len, diag, lo):
    i = torch.arange(n_rows).unsqueeze(1) + q_off
    j = torch.arange(kv_len).unsqueeze(0)
    m = torch.ones(n_rows, kv_len, dtype=torch.bool)
    if diag < DIAG_FULL:
        m &= j <= i + diag
    if lo > LO_NONE:
        m &= j >= i + lo
    return m


class FakeExt:
    def __init__(self):
        self.calls = []

    # ------------------------------------------------------------------ forward
    def _fwd(self, q, k, v, items, segs, seg_lo, out, lse, scale, sqk=None, sv=None):
        hq, hkv = q.shape[1], k.shape[1]
        rep = hq // hkv
        qf, kf, vf = q.float(), k.float(), v.float()
        segs = segs.tolist()
        for q_row0, n_rows, q_off, seg_begin, seg_count, *_ in items.tolist():
            scores, vals = [], []
            for si in range(seg_begin, seg_begin + seg_count):
                kv_row0, kv_len, diag, _flag = segs[si]
                lo = LO_NONE if seg_lo is None else int(seg_lo[si])
                m = _visible(n_rows, q_off, kv_len, diag, lo)  # (n, kv_len)
                kk = kf[kv_row0:kv_row0 + kv_len].repeat_interleave(rep, dim=1)  # (kv_len, hq, d)
                vv = vf[kv_row0:kv_row0 + kv_len].repeat_interleave(rep, dim=1)
                s = torch.einsum("nhd,khd->hnk", qf[q_row0:q_row0 + n_rows], kk) * scale
                if sqk is not None:
                    s = s * sqk.view(-1, 1, 1)
                scores.append(s.masked_fill(~m.unsqueeze(0), float("-inf")))
                vals.append(vv)
            s = torch.cat(scores, dim=-1)
            vv = torch.cat(vals, dim=0)
            l = torch.logsumexp(s, dim=-1)  # (hq, n)
            p = torch.exp(s - torch.where(torch.isinf(l), torch.zeros_like(l), l).unsqueeze(-1))
            p = torch.where(torch.isinf(s), torch.zeros_like(p), p)
            o = torch.einsum("hnk,khd->nhd", p, vv)
            if sv is not None:
                o = o * sv.repeat_interleave(rep).view(1, -1, 1)
            out[q_row0:q_row0 + n_rows] = o.to(out.dtype)
            lse[:, q_row0:q_row0 + n_rows] = l

    def attn_fwd(self, q, k, v, items, segs, out, lse, lse_S, scale):
        self.calls.append("attn_fwd")
        assert lse_S == q.shape[0]
        self._fwd(q, k, v, items, segs, None, out, lse, scale)

    def attn_fwd_window(self, q, k, v, items, segs, seg_lo, out, lse, lse_S, scale):
        self.calls.append("attn_fwd_window")
        assert seg_lo.numel() == segs.shape[0]
        self._fwd(q, k, v, items, segs, seg_lo.tolist(), out, lse, scale)

    def attn_fwd_fp8(self, q, k, v, items, segs, q_scale, q_block, k_scale, v_scale, kv_block, v_ref, kv_row0, out, lse,
                     lse_S, scale):
        """Contract of the block-scaled fp8 forward: dequantise with the tables, then the plain forward."""
        self.calls.append("attn_fwd_fp8")
        assert q.dtype == torch.float8_e4m3fn and out.dtype == torch.bfloat16
        assert q_scale.shape[1] == q.shape[1] and k_scale.shape[1] == k.shape[1] == v_scale.shape[1]
        assert torch.allclose(v_ref, v_scale.amax(dim=0)) or v_ref.numel() == k.shape[1]

        def deq(x, table, block, row0=0):
            rows = torch.arange(x.shape[0]) + row0
            return x.float() * table[rows // block].unsqueeze(-1)

        self._fwd(deq(q, q_scale, q_block), deq(k, k_scale, kv_block, kv_row0), deq(v, v_scale, kv_block, kv_row0),
                  items, segs, None, out, lse, scale)

    # ------------------------------------------------------------------ backward
    def attn_bwd_delta(self, out, dout, delta, lse_S):
        self.calls.append("attn_bwd_delta")
        delta.copy_((out.float() * dout.float()).sum(-1).transpose(0, 1))

    def _bwd(self, q, dout, k, v, dq, items, qsegs, lse, delta, dk, dv, scale, window):
        hq, hkv = q.shape[1], k.shape[1]
        rep = hq // hkv
        qf, dof, kf, vf = q.float(), dout.float(), k.float(), v.float()
        qsegs = qsegs.tolist()
        for kv_row0, kv_rows, seg_begin, seg_count, *_ in items.tolist():
            kt = kf[kv_row0:kv_row0 + kv_rows].repeat_interleave(rep, dim=1)  # (kr, hq, d)
            vt = vf[kv_row0:kv_row0 + kv_rows].repeat_interleave(rep, dim=1)
            dk_t = torch.zeros(kv_rows, hq, q.shape[2])
            dv_t = torch.zeros(kv_rows, hq, q.shape[2])
            for q_row0, q_len, diag, lo in qsegs[seg_begin:seg_begin + seg_count]:
                rows = slice(q_row0, q_row0 + q_len)
                m = _visible(q_len, 0, kv_rows, diag, lo if window else LO_NONE)
                s = torch.einsum("nhd,khd->hnk", qf[rows], kt) * scale
                lr = lse[:, rows]
                p = torch.exp(s - torch.where(torch.isinf(lr), torch.full_like(lr, float("inf")), lr).unsqueeze(-1))
                p = p.masked_fill(~m.unsqueeze(0), 0.0)
                dv_t += torch.einsum("hnk,nhd->khd", p, dof[rows])
                dp = torch.einsum("nhd,khd->hnk", dof[rows], vt)
                ds = p * (dp - delta[:, rows].unsqueeze(-1)) * scale
                dk_t += torch.einsum("hnk,nhd->khd", ds, qf[rows])
                dq[rows] += torch.einsum("hnk,khd->nhd", ds, kt)
            d = q.shape[2]
            dk[kv_row0:kv_row0 + kv_rows] = dk_t.view(kv_rows, hkv, rep, d).sum(2)  # written, not accumulated
            dv[kv_row0:kv_row0 + kv_rows] = dv_t.view(kv_rows, hkv, rep, d).sum(2)

    def dq_finalize(self, acc, out):
        self.calls.append("dq_finalize")
        out.copy_(acc.to(out.dtype))
        acc.zero_()

    def attn_bwd(self, q, dout, k, v, dq, items, qsegs, lse, delta, dk, dv, lse_S, scale):
        self.calls.append("attn_bwd")
        self._bwd(q, dout, k, v, dq, items, qsegs, lse, delta, dk, dv, scale, False)

    def attn_bwd_window(self, q, dout, k, v, dq, items, qsegs, lse, delta, dk, dv, lse_S, scale):
        self.calls.append("attn_bwd_window")
        self._bwd(q, dout, k, v, dq, items, qsegs, lse, delta, dk, dv, scale, True)


def install():
    """Route the library's launches to a :class:`FakeExt` and make every tensor look kernel-eligible."""
    import os

    from ring_flash_attn_b200.ops import cuda_ext

    fake = FakeExt()
    cuda_ext.load = lambda: fake
    cuda_ext.available_for = lambda t: os.environ.get("RFA_B200_FORCE_TORCH", "0") != "1"
    return fake
