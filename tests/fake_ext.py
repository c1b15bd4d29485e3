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

    # the pieces of the contract that tests/test_kernel_oracle_cpu.py mutates
    def _mask(self, n_rows, q_off, kv_len, diag, lo):
        return _visible(n_rows, q_off, kv_len, diag, lo)

    def _kv_heads(self, x, rep):  # query head h reads kv head h // rep
        return x.repeat_interleave(rep, dim=1)

    def _p_for_pv(self, p, dtype):  # P as the P V product sees it
        return p

    def _group_sum(self, x, hkv, rep):  # dK / dV of a kv head: sum over its query heads
        return x.view(x.shape[0], hkv, rep, x.shape[2]).sum(2)

    def _accumulate(self, acc, x, dtype):  # a key tile's dK / dV after one more query segment
        return acc + x

    def _dq_part(self, x, q_row0, kv_row0):  # the dQ contribution of one key tile to rows q_row0 ..
        return x

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
                m = self._mask(n_rows, q_off, kv_len, diag, lo)  # (n, kv_len)
                kk = self._kv_heads(kf[kv_row0:kv_row0 + kv_len], rep)  # (kv_len, hq, d)
                vv = self._kv_heads(vf[kv_row0:kv_row0 + kv_len], rep)
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
            o = torch.einsum("hnk,khd->nhd", self._p_for_pv(p, out.dtype), vv)
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
            kt = self._kv_heads(kf[kv_row0:kv_row0 + kv_rows], rep)  # (kr, hq, d)
            vt = self._kv_heads(vf[kv_row0:kv_row0 + kv_rows], rep)
            dk_t = torch.zeros(kv_rows, hq, q.shape[2])
            dv_t = torch.zeros(kv_rows, hq, q.shape[2])
            for q_row0, q_len, diag, lo in qsegs[seg_begin:seg_begin + seg_count]:
                rows = slice(q_row0, q_row0 + q_len)
                m = self._mask(q_len, 0, kv_rows, diag, lo if window else LO_NONE)
                s = torch.einsum("nhd,khd->hnk", qf[rows], kt) * scale
                lr = lse[:, rows]
                p = torch.exp(s - torch.where(torch.isinf(lr), torch.full_like(lr, float("inf")), lr).unsqueeze(-1))
                p = p.masked_fill(~m.unsqueeze(0), 0.0)
                dv_t = self._accumulate(dv_t, torch.einsum("hnk,nhd->khd", self._p_for_pv(p, q.dtype), dof[rows]),
                                        q.dtype)
                dp = torch.einsum("nhd,khd->hnk", dof[rows], vt)
                ds = p * (dp - delta[:, rows].unsqueeze(-1)) * scale
                dk_t = self._accumulate(dk_t, torch.einsum("hnk,nhd->khd", ds, qf[rows]), q.dtype)
                dq[rows] += self._dq_part(torch.einsum("hnk,khd->nhd", ds, kt), q_row0, kv_row0)
            dk[kv_row0:kv_row0 + kv_rows] = self._group_sum(dk_t, hkv, rep)  # written, not accumulated
            dv[kv_row0:kv_row0 + kv_rows] = self._group_sum(dv_t, hkv, rep)

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


class FakeDecodeExt:
    """The contract of the split-KV decode kernels (``decode_fwd``, ``decode_combine``, ``csrc/decode_sm90.cu``) in
    torch, independently of ``parallel.decode._dense_decode``: the append (rows past the capacity or outside the pool
    dropped, K rotated, e4m3 quantisation), one fp32 partial per split of ``tiles_per_split`` 128-key tiles in the
    ``(n_splits, rows * Hq * D + Hq * rows)`` layout (out 0 and lse -inf where a split sees no key), the varlen
    tile-slot schedule, and the combine.  Not wired into :func:`install`: route ``cuda_ext.load`` to it directly."""

    def __init__(self):
        self.calls = []

    # ------------------------------------------------------------------ the pieces tests/test_decode_oracle_cpu.py mutates
    def _n_vis(self, t, n_q, causal, appended):  # keys appended by this call that token t sees
        return 0 if not appended else (t + 1 if causal else n_q)

    def _tiles_per_split(self, tiles, n_splits):
        return -(-tiles // n_splits)

    def _kv_head(self, h, group, hkv):  # query head h reads kv head h // G
        return h // group

    def _p_for_pv(self, p, dtype):  # P as the P V product sees it
        return p.to(dtype).float()

    def _k_descale(self, ds, b, kv_head):
        return ds[b, kv_head]

    def _v_descale(self, ds, b, kv_head):
        return ds[b, kv_head]

    def _q_position(self, start, t, causal):  # rotary table row of query token t
        return start + t if causal else start

    def _page_row(self, key, page_size):  # row of logical key `key` inside its page
        return key % page_size

    def _carry(self, base, step_tiles):  # tiles before the next 32-sequence step of the varlen prefix sum
        return base + step_tiles

    def _empty_lse(self):
        return float("-inf")

    def _finish_lse(self, lse):
        return lse

    def _combine_parts(self, parts):
        return parts

    # ------------------------------------------------------------------ helpers
    def _slots(self, tiles, n_slots):
        """Tile slot -> (sequence, row tile) as ``varlen_tile`` maps it, 32 sequences per step."""
        out = {}
        for slot in range(n_slots):
            base = 0
            for c in range(0, len(tiles), 32):
                incl = 0
                for i, n in enumerate(tiles[c:c + 32]):
                    incl += n
                    if base + incl - n <= slot < base + incl:
                        out[slot] = (c + i, slot - (base + incl - n))
                        break
                if slot in out:
                    break
                base = self._carry(base, incl)
        return out

    def decode_fwd(self, q, k_cache, v_cache, seqlens, k_new, v_new, causal, scale, part, block_table, k_descale,
                   v_descale, cu_seqlens_q, max_seqlen_q, rotary_cos, rotary_sin, rotary_seqlens, rotary_interleaved):
        from ring_flash_attn_b200.parallel.decode import apply_rotary, quantize_e4m3, tile_slots

        self.calls.append("decode_fwd")
        # the binding's check: the kernel stores out as float2, so every split's partial starts 8-byte aligned
        assert part.dtype == torch.float32 and part.stride(1) == 1 and part.stride(0) % 2 == 0, \
            "decode_fwd: every split's partial must start 8-byte aligned"
        varlen = cu_seqlens_q is not None
        nb = seqlens.numel()
        if varlen:
            rows, hq, d = q.shape
            sq = max_seqlen_q
            cu = [min(max(x, 0), rows) for x in cu_seqlens_q.tolist()]  # clamped as q_rows() does
            spans = [(cu[i], min(max(cu[i + 1] - cu[i], 0), sq)) for i in range(nb)]
        else:
            _, sq, hq, d = q.shape
            rows = nb * sq
            spans = [(i * sq, sq) for i in range(nb)]
            q = q.reshape(rows, hq, d)
            if k_new is not None:
                k_new, v_new = k_new.reshape(rows, *k_new.shape[2:]), v_new.reshape(rows, *v_new.shape[2:])
        hkv = k_cache.shape[2]
        group = hq // hkv
        paged = block_table is not None
        ps = k_cache.shape[1] if paged else 0
        n_pages = k_cache.shape[0]
        s_cap = block_table.shape[1] * ps if paged else k_cache.shape[1]
        fp8 = k_cache.dtype == torch.float8_e4m3fn
        lens = seqlens.tolist()
        table = block_table.tolist() if paged else None
        rot = rotary_cos is not None
        seqlen_ro = rotary_cos.shape[0] if rot else 0
        rs = rotary_seqlens.tolist() if rot else None

        def clamp_pos(x):
            return min(max(x, 0), seqlen_ro - 1)

        def loc(b, row):  # (page or sequence, row) of logical row `row`, None when outside the pool
            if not paged:
                return b, row
            page = table[b][row // ps]
            return (page, self._page_row(row, ps)) if 0 <= page < n_pages else None

        # ---- the append
        if k_new is not None:
            for b, (lo, cnt) in enumerate(spans):
                for t in range(cnt):
                    row = lens[b] + t
                    at = loc(b, row) if 0 <= row < s_cap else None
                    if at is None:
                        continue
                    kx, vx = k_new[lo + t], v_new[lo + t]
                    if rot:
                        pos = torch.tensor([clamp_pos(rs[b] + t)])
                        kx = apply_rotary(kx[None], rotary_cos, rotary_sin, pos, rotary_interleaved)[0]
                    if fp8:
                        kx, vx = quantize_e4m3(kx, k_descale[b]), quantize_e4m3(vx, v_descale[b])
                    k_cache[at] = kx
                    v_cache[at] = vx

        # ---- per-split partials
        n_splits = part.shape[0]
        tiles = max(1, -(-s_cap // 128))
        span = self._tiles_per_split(tiles, n_splits) * 128
        part.fill_(float("nan"))  # what an unwritten row of torch.empty may hold
        n_out = rows * hq * d
        out_p = part[:, :n_out].view(n_splits, rows, hq, d)
        lse_p = part[:, n_out:]
        t2 = torch.tensor(scale * 1.4426950408889634, dtype=torch.float32)
        row_tiles = [-(-n * group // 64) for _, n in spans]
        if varlen:
            work = self._slots(row_tiles, tile_slots(nb, rows, sq, hq, hkv)).values()
        else:
            work = [(b, tile) for b in range(nb) for tile in range(row_tiles[b])]
        for b, tile in work:
            lo, cnt = spans[b]
            n = min(max(lens[b], 0), s_cap)
            packed_rows = range(tile * 64, min(tile * 64 + 64, cnt * group))
            if not packed_rows:
                continue
            for kvh in range(hkv):
                ts = [pr // group for pr in packed_rows]
                hs = [kvh * group + pr % group for pr in packed_rows]
                row_idx, head_idx = torch.tensor([lo + t for t in ts]), torch.tensor(hs)
                # lse of (head, t): (B, Hq, Sq) uniform, (Hq, total_q) varlen
                lse_idx = head_idx * rows + row_idx if varlen else (b * hq + head_idx) * sq + torch.tensor(ts)
                lim = torch.tensor([min(n + self._n_vis(t, cnt, causal, k_new is not None), s_cap) for t in ts])
                kmax = int(lim.max())
                qr = q[[lo + t for t in ts], hs]  # (r, D)
                if rot:
                    pos = torch.tensor([clamp_pos(self._q_position(rs[b], t, causal)) for t in ts])
                    qr = apply_rotary(qr[:, None], rotary_cos, rotary_sin, pos, rotary_interleaved)[:, 0]
                kvs = [self._kv_head(h, group, hkv) for h in hs]
                locs = [loc(b, j) for j in range(kmax)]
                assert all(x is not None for x in locs), "a visible key's page is outside the pool"
                idx = tuple(torch.tensor(list(c), dtype=torch.long) for c in zip(*locs)) if locs else None
                kk = torch.zeros(kmax, len(hs), d)
                vv = torch.zeros(kmax, len(hs), d)
                if kmax:
                    kk = k_cache[idx][:, kvs].to(q.dtype).float()  # (keys, r, D); e4m3 widens exactly
                    vv = v_cache[idx][:, kvs].to(q.dtype).float()
                s = torch.einsum("rd,jrd->rj", qr.float(), kk)
                s = s.masked_fill(torch.arange(kmax)[None] >= lim[:, None], float("-inf"))
                tt = t2 * torch.stack([self._k_descale(k_descale, b, kvh) for _ in hs]) if fp8 else t2
                tt = tt.view(-1, 1) if fp8 else tt
                vd = torch.stack([self._v_descale(v_descale, b, kvh) for _ in hs]) if fp8 else None
                for sp in range(n_splits):
                    a, e = sp * span, min((sp + 1) * span, kmax)
                    o = torch.zeros(len(hs), d)
                    lse = torch.full((len(hs),), self._empty_lse())
                    if a < e:
                        ss = s[:, a:e]
                        mx = ss.amax(dim=1, keepdim=True)
                        empty = torch.isinf(mx)
                        m2 = torch.where(empty, torch.zeros_like(mx), mx * tt)
                        p = torch.exp2(ss * tt - m2)
                        l = p.sum(dim=1, keepdim=True)
                        o = torch.einsum("rj,jrd->rd", self._p_for_pv(p, q.dtype), vv[a:e])
                        inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
                        if fp8:
                            inv = inv * vd.view(-1, 1)
                        o = o * inv
                        lse = torch.where(empty[:, 0], lse, (m2 + torch.log2(l))[:, 0] * 0.6931471805599453)
                    out_p[sp, row_idx, head_idx] = o
                    lse_p[sp, lse_idx] = self._finish_lse(lse)

    def decode_combine(self, parts, out, lse):
        self.calls.append("decode_combine")
        b, sq, hq, d = out.shape
        parts = self._combine_parts(parts)
        n_out = b * sq * hq * d
        o = parts[:, :n_out].view(-1, b, sq, hq, d)
        l = parts[:, n_out:].view(-1, b, hq, sq).permute(0, 1, 3, 2).unsqueeze(-1)  # (P, B, Sq, Hq, 1)
        if parts.shape[0] == 0:  # nothing to merge: no key seen
            out.zero_()
            lse.fill_(float("-inf"))
            return
        skip = torch.isneginf(l)
        mx = l.amax(dim=0)
        ok = ~torch.isneginf(mx)
        mx0 = torch.where(ok, mx, torch.zeros_like(mx))
        tot = torch.where(skip, torch.zeros_like(l), torch.exp(l - mx0)).sum(dim=0)
        lc = torch.where(ok, mx + torch.log(tot), torch.full_like(mx, float("-inf")))
        w = torch.exp(l - torch.where(ok, lc, torch.zeros_like(lc)))
        acc = torch.where(skip | ~ok, torch.zeros_like(o), w * o).sum(dim=0)  # a skipped partial's out is not read
        out.copy_(acc.to(out.dtype))
        lse.view(b, hq, sq).copy_(lc[..., 0].permute(0, 2, 1))


def install():
    """Route the library's launches to a :class:`FakeExt` and make every tensor look kernel-eligible."""
    import os

    from ring_flash_attn_b200.ops import cuda_ext

    fake = FakeExt()
    cuda_ext.load = lambda: fake
    cuda_ext.available_for = lambda t: os.environ.get("RFA_B200_FORCE_TORCH", "0") != "1"
    return fake
