"""The sm_90a split-KV decode kernel with fp8 (e4m3) queries over e4m3 caches (``q_descale``), at head_dim 64 and
128: the fp64 oracle over the geometries and value regimes of ``tests/decode_oracle.py`` (appends of bf16 and of
pre-quantised e4m3 k / v), bitwise relations (power-of-two q_descale against softmax_scale, paged against contiguous,
varlen against uniform, NaN past the valid rows), the append bytes, CUDA-graph replay with new lengths and
q_descale, and the cross-rank merge on two GPUs."""
import dataclasses

import pytest
import torch

import decode_oracle as DO
import decode_q8 as Q8
from dist_utils import run_distributed
from ring_flash_attn_b200.parallel import decode as dec
from test_gpu_decode_fp8 import bytes_of

pytestmark = pytest.mark.gpu

HEAD_DIMS = [64, 128]
NO_ROTARY = [g.name for g in DO.GEOMETRIES if g.rotary is None]
APPENDING = [g.name for g in DO.GEOMETRIES if g.rotary is None and g.append]


@pytest.fixture(autouse=True)
def _exact_fp32_matmul():
    """The precision-matched reference needs true fp32 GEMMs."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("d", HEAD_DIMS)
def test_q8_sweep(d):
    """Every geometry without rotary and every value regime, appending bf16 k / v; then every appending geometry with
    pre-quantised e4m3 k / v."""
    for name, regime in DO.sweep_cases(NO_ROTARY):
        Q8.run_q8(DO.geometry(name), d, regime, "cuda")
    for name in APPENDING:
        Q8.run_q8(DO.geometry(name), d, "randn", "cuda", append_kind="e4m3")


def _inputs(case, d, seed=0):
    inp = DO.build_inputs(dataclasses.replace(case, fp8=True), torch.bfloat16, d, "randn", "cuda", seed)
    q8, qd, _ = Q8.quantise_q(inp)
    return inp, q8, qd


def _call(inp, q8, qd, caches=None, splits=4, scale=None, append="bf16", **over):
    """kernel_decode on (copies of) the case's caches; returns (out, lse, k_cache, v_cache)."""
    case = inp.case
    kc, vc = caches if caches is not None else (inp.k_cache.clone(), inp.v_cache.clone())
    src = dataclasses.replace(inp, q=q8)
    if append == "e4m3":
        src = dataclasses.replace(src, k_new=inp.stored_k, v_new=inp.stored_v)
    q, k, v = DO.call_views(src, case.append)
    kw = DO.call_kwargs(inp)
    kw.update(over)
    out, lse = dec.kernel_decode(q, kc, vc, inp.seqlens, k, v, case.causal,
                                 inp.d ** -0.5 if scale is None else scale, splits=splits, q_descale=qd, **kw)
    return out, lse, kc, vc


@pytest.mark.parametrize("d", HEAD_DIMS)
def test_power_of_two_q_descale_is_softmax_scale(d):
    inp, q8, _ = _inputs(DO.geometry("splits_default"), d)
    for a in (-3, 2):
        p2 = torch.full((inp.case.b, inp.case.hkv), 2.0 ** a, device="cuda")
        out, lse, _, _ = _call(inp, q8, p2)
        ref_out, ref_lse, _, _ = _call(inp, q8, torch.ones_like(p2), scale=d ** -0.5 * 2.0 ** a)
        assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), a


@pytest.mark.parametrize("append", ["bf16", "e4m3"])
@pytest.mark.parametrize("name", ["paged16", "paged128", "varlen44_paged32"])
@pytest.mark.parametrize("d", HEAD_DIMS)
def test_paged_equals_contiguous(d, name, append):
    paged = DO.geometry(name)
    flat = dataclasses.replace(paged, layout="contiguous", page_size=0)
    inp_p, q8, qd = _inputs(paged, d)
    inp_c, q8c, qdc = _inputs(flat, d)
    assert torch.equal(bytes_of(inp_p.kc0), bytes_of(inp_c.kc0)) and torch.equal(q8.view(torch.uint8),
                                                                                q8c.view(torch.uint8))
    out_p, lse_p, kp, vp = _call(inp_p, q8, qd, append=append)
    out_c, lse_c, kc, vc = _call(inp_c, q8c, qdc, append=append)
    assert torch.equal(out_p, out_c) and torch.equal(lse_p, lse_c)
    # the appended rows reached the same logical cache
    rows = [min(n + c, paged.s_cap) for n, c in zip(inp_p.lens, paged.counts)]
    table = inp_p.table.tolist()
    ps = paged.page_size
    for b, n in enumerate(rows):
        for j in range(n):
            pg = table[b][j // ps]
            assert torch.equal(kp[pg, j % ps].view(torch.uint8), kc[b, j].view(torch.uint8)), (b, j)
            assert torch.equal(vp[pg, j % ps].view(torch.uint8), vc[b, j].view(torch.uint8)), (b, j)


@pytest.mark.parametrize("d", HEAD_DIMS)
def test_varlen_equal_counts_equals_uniform(d):
    uni = DO.Case("uni", (3,) * 5, (700, 0, 129, 300, 1000), 1024, hq=16, hkv=2)
    var = dataclasses.replace(uni, name="var", varlen=True)
    inp_u, q8u, qdu = _inputs(uni, d)
    inp_v, q8v, qdv = _inputs(var, d)
    out_u, lse_u, ku, _ = _call(inp_u, q8u, qdu, splits=3)
    out_v, lse_v, kv, _ = _call(inp_v, q8v, qdv, splits=3)
    got_o, got_l = DO.packed(uni, out_u, lse_u)
    assert torch.equal(got_o, out_v) and torch.equal(got_l, lse_v)
    assert torch.equal(bytes_of(ku), bytes_of(kv))


@pytest.mark.parametrize("append", ["bf16", "e4m3"])
@pytest.mark.parametrize("d", HEAD_DIMS)
def test_varlen_sequence_equals_its_uniform_call(d, append):
    var = DO.Case("var", (3, 0, 1, 5, 2), (350, 9, 0, 200, 640), 700, hq=8, hkv=2, varlen=True)
    inp, q8, qd = _inputs(var, d)
    out, lse, _, _ = _call(inp, q8, qd, splits=3, append=append)
    for b, (lo, n) in enumerate(DO.spans(var)):
        if n == 0:
            continue
        one = dataclasses.replace(var, name="one", counts=(n,), seqlens=(var.seqlens[b],), varlen=False)
        sub = dataclasses.replace(inp, case=one, q=inp.q[lo:lo + n], k_new=inp.k_new[lo:lo + n],
                                  v_new=inp.v_new[lo:lo + n], stored_k=inp.stored_k[lo:lo + n],
                                  stored_v=inp.stored_v[lo:lo + n], seqlens=inp.seqlens[b:b + 1],
                                  k_descale=inp.k_descale[b:b + 1], v_descale=inp.v_descale[b:b + 1])
        caches = (inp.k_cache[b:b + 1].clone(), inp.v_cache[b:b + 1].clone())
        o1, l1, _, _ = _call(sub, q8[lo:lo + n], qd[b:b + 1], caches=caches, splits=3, append=append)
        assert torch.equal(o1[0], out[lo:lo + n]) and torch.equal(l1[0], lse[:, lo:lo + n]), b


@pytest.mark.parametrize("d", HEAD_DIMS)
def test_nan_past_valid_rows_is_never_read(d):
    case = DO.geometry("split_edge_by_append")
    inp, q8, qd = _inputs(case, d)
    clean_k, clean_v = inp.k_cache.clone(), inp.v_cache.clone()
    for b, n in enumerate(inp.lens):  # zero bytes where build_inputs left e4m3 NaN
        clean_k.view(torch.uint8)[b, n:] = 0
        clean_v.view(torch.uint8)[b, n:] = 0
    for append in ("bf16", "e4m3"):
        out, lse, _, _ = _call(inp, q8, qd, append=append)
        ref_out, ref_lse, _, _ = _call(inp, q8, qd, caches=(clean_k.clone(), clean_v.clone()), append=append)
        assert torch.isfinite(out).all()
        assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), append


@pytest.mark.parametrize("d", HEAD_DIMS)
def test_append_bytes(d):
    """e4m3 k / v are stored as they are; bf16 k / v exactly as the bf16-q e4m3 append stores them."""
    case = DO.geometry("saturating_append")
    inp, q8, qd = _inputs(case, d)
    _, _, k8, v8 = _call(inp, q8, qd, append="e4m3")
    want_k, want_v = DO.expected_caches(inp, inp.k_cache, inp.v_cache, True)
    assert torch.equal(bytes_of(k8), bytes_of(want_k)) and torch.equal(bytes_of(v8), bytes_of(want_v))
    _, _, kq, vq = _call(inp, q8, qd, append="bf16")
    kb, vb = inp.k_cache.clone(), inp.v_cache.clone()
    q, k, v = DO.call_views(inp, True)
    dec.kernel_decode(q, kb, vb, inp.seqlens, k, v, case.causal, d ** -0.5, splits=4, **DO.call_kwargs(inp))
    assert torch.equal(bytes_of(kq), bytes_of(kb)) and torch.equal(bytes_of(vq), bytes_of(vb))


def test_cuda_graph_replay_with_new_lengths_and_q_descale():
    case = DO.Case("graph", (2,) * 4, (1000, 2500, 7, 0), 3008, hq=32, hkv=8)
    inp, q8, qd = _inputs(case, 128)
    kc, vc = inp.k_cache.clone(), inp.v_cache.clone()
    for c in (kc, vc):  # finite everywhere: the replays move the valid lengths past the rows build_inputs left NaN
        raw = c.view(torch.uint8)
        raw[(raw & 0x7F) == 0x7F] = 0
    q, k, v = DO.call_views(dataclasses.replace(inp, q=q8), True)
    sl = inp.seqlens.clone()
    qd_buf = qd.clone()
    kw = dict(splits=4, k_descale=inp.k_descale, v_descale=inp.v_descale, q_descale=qd_buf)

    def step(kc_, vc_):
        return dec.kernel_decode(q, kc_, vc_, sl, k, v, True, 128 ** -0.5, **kw)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(kc.clone(), vc.clone())  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, lse = step(kc, vc)
    for lens_now, factor in (([1000, 2500, 7, 0], 1.0), ([1200, 1, 0, 3000], 0.75), ([0, 2999, 64, 5], 1.5)):
        sl.copy_(torch.tensor(lens_now, dtype=torch.int32))
        qd_buf.copy_(qd * factor)
        ek, ev = kc.clone(), vc.clone()
        g.replay()
        want_out, want_lse = step(ek, ev)
        torch.cuda.synchronize()
        assert torch.equal(out, want_out) and torch.equal(lse, want_lse), lens_now
        assert torch.equal(bytes_of(kc), bytes_of(ek)) and torch.equal(bytes_of(vc), bytes_of(ev)), lens_now


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_combine_matches_oracle():
    run_distributed(Q8.run_two_ranks_q8, 2, "cuda", backend="nccl")
