"""Decode step against a long KV cache: the sm_90a split-KV kernel vs torch SDPA (``enable_gqa=True``) on the same
local shard, alternating in one run.

One JSON line per (batch, cache length): device-timed microseconds per call, the K + V bytes the call must read, the
achieved rate and its share of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s; a data-sheet figure, not a measured
peak), with the card name and power limit.  Under ``torchrun`` (world > 1) every rank holds a shard of that length and
the line also reports the all-gather + combine time of the cross-rank merge.  With ``--page-size N`` every
configuration also times the kernel on a paged copy of the same cache (pages in a seeded random order, one block
table per sequence) in the same alternating loop, and reports whether its output is bitwise the contiguous one.
With ``--kv-dtype e4m3`` every configuration also times the kernel over an e4m3 copy of the cache (quantised with
per-(sequence, kv head) descales; paged too with ``--page-size``) in the same loop, and reports its bytes, rate,
speed-up over the bf16 kernel, whether its output at unit descales is bitwise the bf16 kernel's on the widened cache,
and its largest difference from the bf16 output (the quantisation error, for information).
With ``--q-dtype e4m3`` (which needs ``--kv-dtype e4m3``) the loop gains a third arm: the fp8-query kernel (an e4m3
query with per-(sequence, kv head) ``q_descale``, Q K^T as an e4m3 wgmma) over the same e4m3 cache (paged too with
``--page-size``); the line reports its time, its speed-up over the bf16 arm and over the bf16-query e4m3-cache arm,
and its largest difference from the bf16 output (for information).
With ``--mixed-chunk C`` every configuration also times, in the same loop, a varlen call (``cu_seqlens_q``) where
sequence 0 brings C new tokens and the others 1, the uniform call padded to Sq = C (what a caller without varlen
must do) and the uniform Sq = 1 call (the pure-decode floor), with the K + V bytes the varlen and padded calls stream
(every 64-row tile streams its sequence's shard).
With ``--rotary`` every configuration also times, in the same loop, a RoPE decode step that appends the new k / v
(the shard then holds the cache length): the fused call (``rotary_cos`` / ``rotary_sin``, non-interleaved, rotary_dim
= head_dim), the same step done without it (``apply_rotary`` on q and k with torch ops, then a plain call), and the
plain call alone; and reports whether the fused and unfused outputs are bitwise equal.
With ``--cache-slots N`` every configuration also times, in the same loop, an appending step over a pool of N cache
slots (each of the cache length) where the B sequences use a seeded random subset of slots (``cache_batch_idx``),
the same step on a B-slot cache with the same contents, and what a caller without ``cache_batch_idx`` must do:
``index_select`` the B slots out of the pool, the plain call, and ``index_copy_`` them back; and reports whether
the slot and plain outputs are bitwise equal.  With ``--leftpad P`` it also times a call whose sequences have P
pad rows below their keys (``cache_leftpad``) against the plain call on the same number of valid rows.  Both arms run
over the cache and query dtypes that ``--kv-dtype`` / ``--q-dtype`` select.
With ``--shared-prefix L --samples n`` the run times shared-prefix decoding instead: P prompts (``--prompts``) of L
tokens per rank, n samples each, every sample with its own ``--suffix`` rows and one appended token per call, in four
arms with the same contents, alternating in one loop: the prefix call (``prefix_k_cache`` / ``prefix_v_cache``), the
prompt copied into each sample's contiguous cache ahead of its suffix (a plain call), paged caches of
``--prefix-page``-row pages (128 by default) whose block tables share the prompt's pages, and the paged prefix call on
that same pool (``prefix_block_table`` names the prompt's pages, ``block_table`` each sample's own).  Each line reports
the HBM bytes each arm must read (from shapes), the largest difference between the arms' outputs, whether the paged
prefix call's out / lse are bitwise the prefix call's, and the card's name, power limit and maximum SM clock (read in
one ``nvidia-smi`` query).  ``--kv-dtype e4m3`` runs the four arms over e4m3 caches with one descale per kv head.
With ``--tree W1,W2,...`` the run times speculative-tree verification instead: a full draft tree in which every node
at depth i has Wi children (plus the root; ``4,2,2,1`` has 45 nodes and 16 leaves), one per sequence, against caches
of ``--cache`` tokens, in three arms alternating in one loop, each appending its tokens: the tree call (``tree_mask``,
Sq = nodes), the causal chain call of the same shape (what the mask costs), and one causal call per root-to-leaf
path (what a caller without ``tree_mask`` must do).  Each line reports the node and leaf counts, the K + V bytes each
arm streams (every 64-row tile of a call streams its sequence's shard), the largest difference between a node's row
in the tree call and the same node's row in a per-path call, and the card's name, power limit and maximum SM clock.

    python benchmark/bench_decode.py                      # B in {1, 8}, caches of 32K..512K tokens per rank
    python benchmark/bench_decode.py --page-size 16       # also the paged kernel, pages of 16 rows
    python benchmark/bench_decode.py --kv-dtype e4m3      # also the fp8-cache kernel
    python benchmark/bench_decode.py --kv-dtype e4m3 --q-dtype e4m3   # and the fp8-query kernel
    python benchmark/bench_decode.py --mixed-chunk 64     # also a ragged batch: one 64-token chunk + decodes
    python benchmark/bench_decode.py --rotary             # also the fused RoPE step against the unfused one
    python benchmark/bench_decode.py --cache 32768 --cache-slots 16   # also a slot pool against gather / scatter
    python benchmark/bench_decode.py --leftpad 1000       # also a left-padded call against the plain one
    torchrun --nproc-per-node 2 benchmark/bench_decode.py
    python benchmark/bench_decode.py --shared-prefix 32768 131072 --samples 4 16   # one prompt, n samples
    python benchmark/bench_decode.py --shared-prefix 32768 --prefix-page 16        # the paged arms in pages of 16
    python benchmark/bench_decode.py --tree 4,2,2,1       # a 45-node draft tree: tree vs chain vs per-path calls
    python benchmark/bench_decode.py --dry-run            # shapes and byte counts only (no GPU)
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ring_flash_attn_b200.parallel import decode as dec  # noqa: E402

HBM_DATASHEET_BPS = 3.35e12  # H100 SXM data sheet, HBM3


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--cache", type=int, nargs="+", default=[32768, 131072, 524288], help="tokens per rank")
    ap.add_argument("--sq", type=int, default=1)
    ap.add_argument("--hq", type=int, default=32)
    ap.add_argument("--hkv", type=int, default=8)
    ap.add_argument("--head-dim", type=int, default=128)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--sm-count", type=int, default=132, help="used by --dry-run only")
    ap.add_argument("--page-size", type=int, default=None, help="also time a paged cache with pages of N rows")
    ap.add_argument("--kv-dtype", choices=("bf16", "e4m3"), default="bf16",
                    help="e4m3: also time an fp8 (e4m3) cache with per-head descales")
    ap.add_argument("--q-dtype", choices=("bf16", "e4m3"), default="bf16",
                    help="e4m3: also time fp8 (e4m3) queries over the e4m3 cache (needs --kv-dtype e4m3)")
    ap.add_argument("--mixed-chunk", type=int, default=None, metavar="C",
                    help="also time a varlen batch (sequence 0 brings C tokens, the others 1) against the uniform "
                         "call padded to Sq = C and the uniform Sq = 1 call")
    ap.add_argument("--rotary", action="store_true",
                    help="also time a RoPE step: the fused call, the torch rotation + a plain call, the plain call")
    ap.add_argument("--cache-slots", type=int, default=None, metavar="N",
                    help="also time a step over an N-slot cache pool (cache_batch_idx) against the plain call and "
                         "the index_select / call / index_copy_ workaround")
    ap.add_argument("--leftpad", type=int, default=None, metavar="P",
                    help="also time a call with P pad rows per sequence (cache_leftpad) against the plain call on "
                         "the same number of valid rows")
    ap.add_argument("--shared-prefix", type=int, nargs="+", default=None, metavar="L",
                    help="time shared-prefix decoding instead: prompts of L tokens per rank (see --samples)")
    ap.add_argument("--samples", type=int, nargs="+", default=[4, 16], help="samples per prompt (--shared-prefix)")
    ap.add_argument("--prompts", type=int, nargs="+", default=[1], help="prompts P per call (--shared-prefix)")
    ap.add_argument("--suffix", type=int, default=256, help="each sample's own cached rows (--shared-prefix)")
    ap.add_argument("--prefix-page", type=int, default=PREFIX_PAGE,
                    help="rows per page of the paged and paged-prefix arms (--shared-prefix)")
    ap.add_argument("--tree", type=str, default=None, metavar="W1,W2,...",
                    help="time tree verification instead: a full tree with Wi children per node at depth i")
    ap.add_argument("--dry-run", action="store_true")
    args = ap.parse_args(argv)
    if args.tree is not None:
        try:
            args.tree = [int(x) for x in args.tree.split(",")]
        except ValueError:
            ap.error("--tree takes comma-separated positive ints, e.g. 4,2,2,1")
        if not args.tree or min(args.tree) < 1 or len(tree_parents(args.tree)) > dec.MAX_TREE_TOKENS:
            ap.error(f"--tree needs positive widths and at most {dec.MAX_TREE_TOKENS} nodes")
    if args.shared_prefix is not None and (min(args.shared_prefix) < 1 or args.suffix < 1 or min(args.samples) < 1
                                           or min(args.prompts) < 1):
        ap.error("--shared-prefix, --samples, --prompts and --suffix must be positive")
    if args.shared_prefix is not None and not dec._valid_page_size(args.prefix_page):
        ap.error("--prefix-page must be 16, 32, 64 or a positive multiple of 128")
    if args.shared_prefix is not None and min(x % args.prefix_page for x in args.shared_prefix) != 0:
        ap.error("--shared-prefix must be a multiple of --prefix-page for the paged arms")
    if args.cache_slots is not None and args.cache_slots < max(args.batch):
        ap.error("--cache-slots must be at least the largest --batch (the sequences use distinct slots)")
    if args.leftpad is not None and not 0 <= args.leftpad < min(args.cache):
        ap.error("--leftpad must be in [0, the smallest --cache)")
    if args.q_dtype == "e4m3" and args.kv_dtype != "e4m3":
        ap.error("--q-dtype e4m3 needs --kv-dtype e4m3 (fp8 queries run over e4m3 caches only)")
    return args


Q8_FIELDS = ["q8_us", "q8_speedup_vs_bf16", "q8_speedup_vs_fp8", "q8_max_abs_diff_vs_bf16"]


def shapes(args, sm_count):
    """One dict per configuration: shapes, split count and the K + V bytes one call reads (bf16)."""
    for b in args.batch:
        for s in args.cache:
            cfg = dict(batch=b, cache_tokens=s, sq=args.sq, hq=args.hq, hkv=args.hkv, head_dim=args.head_dim,
                       splits=dec.num_splits(b, args.sq, args.hq, args.hkv, s, sm_count),
                       kv_bytes=b * s * args.hkv * args.head_dim * 2 * 2)
            if args.page_size:
                cfg.update(page_size=args.page_size, block_table_bytes=b * -(-s // args.page_size) * 4)
            if args.kv_dtype == "e4m3":  # one byte per cached element
                cfg.update(kv_dtype="e4m3", fp8_kv_bytes=cfg["kv_bytes"] // 2)
            if args.q_dtype == "e4m3":  # the fields the timed run adds
                cfg.update(q_dtype="e4m3", q8_fields=Q8_FIELDS)
            if args.mixed_chunk:
                c, g = args.mixed_chunk, args.hq // args.hkv
                total_q = c + b - 1
                shard = s * args.hkv * args.head_dim * 2 * 2  # one sequence's K + V
                chunk_tiles = -(-c * g // dec.ROWS_PER_CTA)
                # every 64-row tile streams its sequence's shard: the bytes the varlen and padded calls move
                cfg.update(mixed_chunk=c, varlen_total_q=total_q,
                           tile_slots=dec.tile_slots(b, total_q, c, args.hq, args.hkv),
                           varlen_splits=dec.num_splits_varlen(b, total_q, c, args.hq, args.hkv, s, sm_count),
                           padded_splits=dec.num_splits(b, c, args.hq, args.hkv, s, sm_count),
                           varlen_kv_bytes=(chunk_tiles + b - 1) * shard, padded_kv_bytes=b * chunk_tiles * shard)
            if args.rotary:  # positions cache_tokens - Sq + t of a table with one row per cached token
                cfg.update(rotary_dim=args.head_dim, rotary_interleaved=False, seqlen_ro=s)
            slot_bytes = cfg["fp8_kv_bytes"] if args.kv_dtype == "e4m3" else cfg["kv_bytes"]  # B slots of K + V
            if args.cache_slots:  # the workaround reads and writes the B slots twice (gather, then scatter)
                cfg.update(cache_slots=args.cache_slots, pool_bytes=slot_bytes // b * args.cache_slots,
                           gather_scatter_bytes=4 * slot_bytes)
            if args.leftpad is not None:
                cfg.update(leftpad=args.leftpad, leftpad_kv_bytes=slot_bytes // s * (s - args.leftpad))
            yield cfg


PREFIX_PAGE = 128  # rows per page of the paged and paged-prefix arms, unless --prefix-page says otherwise


def prefix_shapes(args, sm_count):
    """One dict per shared-prefix configuration: shapes, split counts and the K + V bytes each arm must read."""
    hkv, d, g = args.hkv, args.head_dim, args.hq // args.hkv
    eb = 1 if args.kv_dtype == "e4m3" else 2
    row = hkv * d * 2 * eb  # K + V bytes of one cached token
    for n_prompts in args.prompts:
        for length in args.shared_prefix:
            for n in args.samples:
                b, suf = n_prompts * n, args.suffix
                slots = dec.prefix_tile_slots(n, 1, args.hq, hkv)
                yield dict(shared_prefix=length, samples=n, prompts=n_prompts, batch=b, suffix=suf, sq=1, hq=args.hq,
                           hkv=hkv, head_dim=d, kv_dtype=args.kv_dtype, page_size=args.prefix_page,
                           suffix_splits=dec.num_splits(b, 1, args.hq, hkv, suf, sm_count),
                           prefix_splits=dec.num_splits_prefix(n_prompts, slots, hkv, length, sm_count),
                           plain_splits=dec.num_splits(b, 1, args.hq, hkv, length + suf, sm_count),
                           rows_per_prefix_tile=min(n * g, dec.ROWS_PER_CTA),
                           prefix_bytes=(n_prompts * length + b * suf) * row,
                           copied_bytes=b * (length + suf) * row, paged_bytes=b * (length + suf) * row,
                           paged_prefix_bytes=(n_prompts * length + b * suf) * row)


def card_settings():
    """(name, power limit, max SM clock) of this process's GPU, read in one nvidia-smi query."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], stdout=subprocess.PIPE, text=True, timeout=30)
        name, power, clock = (x.strip() for x in r.stdout.strip().split(","))
    except (OSError, subprocess.SubprocessError, ValueError):
        name, power, clock = torch.cuda.get_device_name(0), "unknown", "unknown"
    return name, power, clock


def shared_prefix_main(args):
    """The four shared-prefix arms, alternating in one loop (see the module docstring)."""
    if args.dry_run:
        for cfg in prefix_shapes(args, args.sm_count):
            print(json.dumps(cfg))
        return
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode.py needs a CUDA device (use --dry-run without one)")
    dev = torch.device("cuda", torch.cuda.current_device())
    name, power, clock = card_settings()
    sm = torch.cuda.get_device_properties(dev).multi_processor_count
    hq, hkv, d = args.hq, args.hkv, args.head_dim
    fp8 = args.kv_dtype == "e4m3"
    for cfg in prefix_shapes(args, sm):
        n_prompts, length, n, b, suf = cfg["prompts"], cfg["shared_prefix"], cfg["samples"], cfg["batch"], cfg["suffix"]
        torch.manual_seed(0)
        q = torch.randn(b, 1, hq, d, device=dev, dtype=torch.bfloat16)
        k_new, v_new = (torch.randn(b, 1, hkv, d, device=dev, dtype=torch.bfloat16) for _ in range(2))
        pk, pv = (torch.randn(n_prompts, length, hkv, d, device=dev, dtype=torch.bfloat16) for _ in range(2))
        sk, sv = (torch.randn(b, suf, hkv, d, device=dev, dtype=torch.bfloat16) for _ in range(2))
        kw, pkw = {}, {}
        if fp8:  # one descale per kv head for prompt and samples alike, so that every arm holds the same contents
            kd = torch.maximum(pk.abs().amax(dim=(0, 1, 3)), sk.abs().amax(dim=(0, 1, 3))).float() / 448
            vd = torch.maximum(pv.abs().amax(dim=(0, 1, 3)), sv.abs().amax(dim=(0, 1, 3))).float() / 448
            pk, sk = (torch.stack([dec.quantize_e4m3(x[i], kd) for i in range(x.shape[0])]) for x in (pk, sk))
            pv, sv = (torch.stack([dec.quantize_e4m3(x[i], vd) for i in range(x.shape[0])]) for x in (pv, sv))
            kw = dict(k_descale=kd.expand(b, hkv).contiguous(), v_descale=vd.expand(b, hkv).contiguous())
            pkw = dict(prefix_k_descale=kd.expand(n_prompts, hkv).contiguous(),
                       prefix_v_descale=vd.expand(n_prompts, hkv).contiguous())
        scale = d ** -0.5
        # every call appends one token at the same row (the last of the suffix), so each arm repeats the same step
        sl_own = torch.full((b,), suf - 1, dtype=torch.int32, device=dev)
        sl_all = sl_own + length
        pl = torch.full((n_prompts,), length, dtype=torch.int32, device=dev)
        owner = torch.arange(b, device=dev) // n

        def raw(x):
            return x.view(torch.uint8)

        # copied: the prompt ahead of each sample's suffix in one contiguous cache
        ck = torch.cat([raw(pk)[owner], raw(sk)], dim=1).view(pk.dtype)
        cv = torch.cat([raw(pv)[owner], raw(sv)], dim=1).view(pv.dtype)
        # paged: the prompt's pages once per prompt, then each sample's own pages; the tables share the prompt pages
        ps = cfg["page_size"]
        p_pages, s_pages = length // ps, -(-suf // ps)

        def pool_of(pre, own):
            rb = d * pre.element_size()  # bytes per (row, kv head)
            pool = torch.zeros((n_prompts * p_pages + b * s_pages, ps, hkv, rb), dtype=torch.uint8, device=dev)
            pool[:n_prompts * p_pages] = raw(pre).reshape(n_prompts * p_pages, ps, hkv, rb)
            padded = torch.zeros((b, s_pages * ps, hkv, rb), dtype=torch.uint8, device=dev)
            padded[:, :suf] = raw(own)
            pool[n_prompts * p_pages:] = padded.view(b * s_pages, ps, hkv, rb)
            return pool.view(pre.dtype)

        gk, gv = pool_of(pk, sk), pool_of(pv, sv)
        prompt_table = torch.arange(n_prompts * p_pages, device=dev, dtype=torch.int32).view(n_prompts, p_pages)
        own_table = (n_prompts * p_pages + torch.arange(b * s_pages, device=dev)).view(b, s_pages).to(torch.int32)
        table = torch.cat([prompt_table[owner], own_table], dim=1)

        def prefix_call():
            return dec.kernel_decode(q, sk, sv, sl_own, k_new, v_new, True, scale, prefix_k_cache=pk,
                                     prefix_v_cache=pv, prefix_seqlens=pl, **kw, **pkw)

        def copied_call():
            return dec.kernel_decode(q, ck, cv, sl_all, k_new, v_new, True, scale, **kw)

        def paged_call():
            return dec.kernel_decode(q, gk, gv, sl_all, k_new, v_new, True, scale, block_table=table, **kw)

        def paged_prefix_call():  # one pool: the prompt's pages by prefix_block_table, the samples' by block_table
            return dec.kernel_decode(q, gk, gv, sl_own, k_new, v_new, True, scale, block_table=own_table,
                                     prefix_k_cache=gk, prefix_v_cache=gv, prefix_block_table=prompt_table,
                                     prefix_seqlens=pl, **kw, **pkw)

        arms = {"prefix": prefix_call, "copied": copied_call, "paged": paged_call, "paged_prefix": paged_prefix_call}
        times = {k: [] for k in arms}
        for _ in range(5):  # alternate them in one run
            for k, fn in arms.items():
                times[k].append(time_us(fn, args.iters, args.warmup))
        res = dict(cfg, card=name, power_limit=power, max_sm_clock=clock)
        for k, ts in times.items():
            us = min(ts)
            res[f"{k}_us"] = round(us, 2)
            res[f"{k}_us_all"] = [round(t, 2) for t in ts]
            res[f"{k}_GBps"] = round(cfg[f"{k}_bytes"] / (us * 1e-6) / 1e9, 1)
        res["prefix_speedup_vs_copied"] = round(res["copied_us"] / res["prefix_us"], 3)
        res["prefix_speedup_vs_paged"] = round(res["paged_us"] / res["prefix_us"], 3)
        res["paged_prefix_speedup_vs_copied"] = round(res["copied_us"] / res["paged_prefix_us"], 3)
        res["paged_prefix_speedup_vs_paged"] = round(res["paged_us"] / res["paged_prefix_us"], 3)
        res["paged_prefix_time_vs_prefix"] = round(res["paged_prefix_us"] / res["prefix_us"], 4)
        results = {k: fn() for k, fn in arms.items()}
        outs = {k: r[0].float() for k, r in results.items()}
        res["max_abs_diff_prefix_vs_copied"] = (outs["prefix"] - outs["copied"]).abs().max().item()
        res["max_abs_diff_paged_vs_copied"] = (outs["paged"] - outs["copied"]).abs().max().item()
        res["max_abs_diff_paged_prefix_vs_copied"] = (outs["paged_prefix"] - outs["copied"]).abs().max().item()
        res["paged_prefix_bitwise_prefix"] = bool(torch.equal(results["paged_prefix"][0], results["prefix"][0])
                                                  and torch.equal(results["paged_prefix"][1], results["prefix"][1]))
        print(json.dumps(res), flush=True)
        del q, k_new, v_new, pk, pv, sk, sv, ck, cv, gk, gv, outs, results
        torch.cuda.empty_cache()


def tree_parents(widths):
    """Parent array (breadth-first, root first) of the full tree with widths[i] children per node at depth i."""
    parents, level = [-1], [0]
    for w in widths:
        nxt = []
        for p in level:
            for _ in range(w):
                parents.append(p)
                nxt.append(len(parents) - 1)
        level = nxt
    return parents


def tree_paths(parents):
    """Root-to-leaf node lists, one per leaf."""
    leaves = sorted(set(range(len(parents))) - set(parents))
    paths = []
    for leaf in leaves:
        path, j = [], leaf
        while j >= 0:
            path.append(j)
            j = parents[j]
        paths.append(path[::-1])
    return paths


def tree_shapes(args, sm_count):
    """One dict per tree configuration: tree size, split counts and the K + V bytes each arm streams."""
    parents = tree_parents(args.tree)
    n, paths = len(parents), tree_paths(parents)
    hkv, d, g = args.hkv, args.head_dim, args.hq // args.hkv
    tiles = -(-n * g // dec.ROWS_PER_CTA)  # 64-row tiles of the tree / chain call
    path_tiles = sum(-(-len(p) * g // dec.ROWS_PER_CTA) for p in paths)
    for b in args.batch:
        for s in args.cache:
            shard = s * hkv * d * 2 * 2  # one sequence's K + V after the append
            yield dict(tree=",".join(map(str, args.tree)), tree_nodes=n, tree_leaves=len(paths),
                       max_depth=len(args.tree), per_path_calls=len(paths), batch=b, cache_tokens=s, hq=args.hq,
                       hkv=hkv, head_dim=d, row_tiles=tiles, tree_splits=dec.num_splits(b, n, args.hq, hkv, s, sm_count),
                       tree_bytes=b * tiles * shard, chain_bytes=b * tiles * shard, per_path_bytes=b * path_tiles * shard)


def tree_main(args):
    """The three tree-verification arms, alternating in one loop (see the module docstring)."""
    if args.dry_run:
        for cfg in tree_shapes(args, args.sm_count):
            print(json.dumps(cfg))
        return
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode.py needs a CUDA device (use --dry-run without one)")
    dev = torch.device("cuda", torch.cuda.current_device())
    name, power, clock = card_settings()
    sm = torch.cuda.get_device_properties(dev).multi_processor_count
    hq, hkv, d = args.hq, args.hkv, args.head_dim
    parents = tree_parents(args.tree)
    n, paths = len(parents), tree_paths(parents)
    anc = torch.zeros(n, n, dtype=torch.bool)
    for i in range(n):
        j = i
        while j >= 0:
            anc[i, j] = True
            j = parents[j]
    for cfg in tree_shapes(args, sm):
        b, s = cfg["batch"], cfg["cache_tokens"]
        torch.manual_seed(0)
        q = torch.randn(b, n, hq, d, device=dev, dtype=torch.bfloat16)
        k_new, v_new = (torch.randn(b, n, hkv, d, device=dev, dtype=torch.bfloat16) for _ in range(2))
        kc, vc = (torch.randn(b, s, hkv, d, device=dev, dtype=torch.bfloat16) for _ in range(2))
        sl = torch.full((b,), s - n, dtype=torch.int32, device=dev)  # the shard holds s rows after the append
        mask = anc.to(dev).expand(b, n, n).contiguous()
        scale = d ** -0.5
        idx = [torch.tensor(p, device=dev) for p in paths]
        pq = [q[:, i].contiguous() for i in idx]
        pk = [k_new[:, i].contiguous() for i in idx]
        pv = [v_new[:, i].contiguous() for i in idx]

        def tree_call():
            return dec.kernel_decode(q, kc, vc, sl, k_new, v_new, True, scale, tree_mask=mask)

        def chain_call():
            return dec.kernel_decode(q, kc, vc, sl, k_new, v_new, True, scale)

        def per_path_call():
            return [dec.kernel_decode(a, kc, vc, sl, x, y, True, scale)[0] for a, x, y in zip(pq, pk, pv)]

        arms = {"tree": tree_call, "chain": chain_call, "per_path": per_path_call}
        times = {k: [] for k in arms}
        order = list(arms)
        for r in range(6):  # alternate them in one run, each arm first in two of the rounds
            for k in order[r % 3:] + order[:r % 3]:
                times[k].append(time_us(arms[k], args.iters, args.warmup))
        res = dict(cfg, card=name, power_limit=power, max_sm_clock=clock)
        for k, ts in times.items():
            us = min(ts)
            res[f"{k}_us"] = round(us, 2)
            res[f"{k}_us_all"] = [round(t, 2) for t in ts]
            res[f"{k}_GBps"] = round(cfg[f"{k}_bytes"] / (us * 1e-6) / 1e9, 1)
        res["tree_speedup_vs_per_path"] = round(res["per_path_us"] / res["tree_us"], 3)
        res["tree_vs_chain"] = round(res["tree_us"] / res["chain_us"], 3)
        tree_out = tree_call()[0].float()
        diff = 0.0
        for i, out in zip(idx, per_path_call()):  # node path[t]'s row in its per-path call
            diff = max(diff, (tree_out[:, i] - out.float()).abs().max().item())
        res["max_abs_diff_tree_vs_per_path"] = diff
        print(json.dumps(res), flush=True)
        del q, k_new, v_new, kc, vc, pq, pk, pv
        torch.cuda.empty_cache()


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], stdout=subprocess.PIPE, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def time_us(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e3 / iters


def main():
    args = parse_args()
    if args.tree is not None:
        tree_main(args)
        return
    if args.shared_prefix is not None:
        shared_prefix_main(args)
        return
    if args.dry_run:
        for cfg in shapes(args, args.sm_count):
            print(json.dumps(cfg))
        return
    import torch.distributed as dist
    import torch.nn.functional as F

    if not torch.cuda.is_available():
        raise SystemExit("bench_decode.py needs a CUDA device (use --dry-run without one)")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
        dist.init_process_group("nccl")
    rank = dist.get_rank() if world > 1 else 0
    dev = torch.device("cuda", torch.cuda.current_device())
    name, power = card()
    sm = torch.cuda.get_device_properties(dev).multi_processor_count
    for cfg in shapes(args, sm):
        b, s, d = cfg["batch"], cfg["cache_tokens"], args.head_dim
        torch.manual_seed(rank)
        q = torch.randn(b, args.sq, args.hq, d, device=dev, dtype=torch.bfloat16)
        kc = torch.randn(b, s, args.hkv, d, device=dev, dtype=torch.bfloat16)
        vc = torch.randn(b, s, args.hkv, d, device=dev, dtype=torch.bfloat16)
        sl = torch.full((b,), s, dtype=torch.int32, device=dev)
        scale = d ** -0.5

        def ours():
            return dec.kernel_decode(q, kc, vc, sl, None, None, True, scale)

        fp8 = args.kv_dtype == "e4m3"
        fp8_res = {}
        if fp8:  # e4m3 copies with per-(sequence, kv head) descales amax / 448, one sequence at a time
            kd = torch.stack([kc[i].abs().amax(dim=(0, 2)).float() for i in range(b)]).clamp(min=1e-12) / 448
            vd = torch.stack([vc[i].abs().amax(dim=(0, 2)).float() for i in range(b)]).clamp(min=1e-12) / 448
            k8 = torch.stack([dec.quantize_e4m3(kc[i], kd[i]) for i in range(b)])
            v8 = torch.stack([dec.quantize_e4m3(vc[i], vd[i]) for i in range(b)])

            def ours_fp8():
                return dec.kernel_decode(q, k8, v8, sl, None, None, True, scale, k_descale=kd, v_descale=vd)

            ones = torch.ones_like(kd)
            wk, wv = k8.to(torch.bfloat16), v8.to(torch.bfloat16)  # the widened cache
            unit = dec.kernel_decode(q, k8, v8, sl, None, None, True, scale, k_descale=ones, v_descale=ones)
            wide = dec.kernel_decode(q, wk, wv, sl, None, None, True, scale)
            fp8_res["fp8_unit_descale_bitwise_equal_bf16"] = all(torch.equal(x, y) for x, y in zip(unit, wide))
            del wk, wv, unit, wide
            fp8_res["fp8_max_abs_diff_vs_bf16"] = (ours_fp8()[0].float() - ours()[0].float()).abs().max().item()

        q8 = args.q_dtype == "e4m3"
        if q8:  # e4m3 queries with per-(sequence, kv head) descales amax / 448, over the same e4m3 cache
            g = args.hq // args.hkv
            qd = q.float().view(b, args.sq, args.hkv, g, d).abs().amax(dim=(1, 3, 4)).clamp(min=1e-12) / 448
            q_e4m3 = (q.float() / qd.repeat_interleave(g, dim=1)[:, None, :, None]).clamp(-448, 448).to(
                torch.float8_e4m3fn)

            def ours_q8():
                return dec.kernel_decode(q_e4m3, k8, v8, sl, None, None, True, scale, k_descale=kd, v_descale=vd,
                                         q_descale=qd)

            fp8_res["q8_max_abs_diff_vs_bf16"] = (ours_q8()[0].float() - ours()[0].float()).abs().max().item()

        if args.page_size:  # the same rows in a pool whose pages are in a seeded random order
            ps = args.page_size
            max_blocks = -(-s // ps)
            perm = torch.randperm(b * max_blocks, generator=torch.Generator().manual_seed(rank)).to(dev)
            table = perm.to(torch.int32).view(b, max_blocks)

            def to_pool(src):
                pool = src.new_zeros(b * max_blocks, ps, args.hkv, d)
                pad = src.new_zeros(b, max_blocks * ps, args.hkv, d)
                pad[:, :s] = src
                pool[perm.long()] = pad.view(b * max_blocks, ps, args.hkv, d)
                return pool

            pk, pv = to_pool(kc), to_pool(vc)

            def paged():
                return dec.kernel_decode(q, pk, pv, sl, None, None, True, scale, block_table=table)

            if fp8:
                p8k, p8v = to_pool(k8.view(torch.uint8)).view(k8.dtype), to_pool(v8.view(torch.uint8)).view(v8.dtype)

                def paged_fp8():
                    return dec.kernel_decode(q, p8k, p8v, sl, None, None, True, scale, block_table=table,
                                             k_descale=kd, v_descale=vd)

                def paged_q8():
                    return dec.kernel_decode(q_e4m3, p8k, p8v, sl, None, None, True, scale, block_table=table,
                                             k_descale=kd, v_descale=vd, q_descale=qd)

        if args.mixed_chunk:  # sequence 0 brings C new tokens, the others 1, over the same caches
            c = args.mixed_chunk
            q_pad = torch.randn(b, c, args.hq, d, device=dev, dtype=torch.bfloat16)
            counts = [c] + [1] * (b - 1)
            q_var = torch.cat([q_pad[i, :n] for i, n in enumerate(counts)])
            cu = torch.tensor([0] + [c + i for i in range(b)], dtype=torch.int32, device=dev)
            q_one = q_pad[:, :1].contiguous()

            def mixed():
                return dec.kernel_decode(q_var, kc, vc, sl, None, None, True, scale, cu_seqlens_q=cu, max_seqlen_q=c)

            def padded():
                return dec.kernel_decode(q_pad, kc, vc, sl, None, None, True, scale)

            def decode_only():
                return dec.kernel_decode(q_one, kc, vc, sl, None, None, True, scale)

        if args.rotary:  # append Sq new tokens at rows [s - Sq, s), rotated at those positions
            k_new = torch.randn(b, args.sq, args.hkv, d, device=dev, dtype=torch.bfloat16)
            v_new = torch.randn_like(k_new)
            sl_app = torch.full((b,), s - args.sq, dtype=torch.int32, device=dev)
            inv = 10000.0 ** (-torch.arange(0, d, 2, dtype=torch.float64, device=dev) / d)
            ang = torch.arange(s, dtype=torch.float64, device=dev)[:, None] * inv[None]
            cos, sin = ang.cos().to(torch.bfloat16), ang.sin().to(torch.bfloat16)
            del ang
            pos = sl_app.long()[:, None] + torch.arange(args.sq, device=dev)[None]  # (B, Sq)

            def rot_fused():
                return dec.kernel_decode(q, kc, vc, sl_app, k_new, v_new, True, scale, rotary_cos=cos,
                                         rotary_sin=sin, rotary_seqlens=sl_app, rotary_interleaved=False)

            def rot_unfused():  # the step without rotary_cos: rotate q and k with torch ops, then a plain call
                qr = dec.apply_rotary(q, cos, sin, pos, False)
                kr = dec.apply_rotary(k_new, cos, sin, pos, False)
                return dec.kernel_decode(qr, kc, vc, sl_app, kr, v_new, True, scale)

            def rot_plain():
                return dec.kernel_decode(q, kc, vc, sl_app, k_new, v_new, True, scale)

        if args.cache_slots or args.leftpad is not None:  # over the cache and query dtypes the flags select
            if q8:
                bq, bk, bv, bkw = q_e4m3, k8, v8, dict(k_descale=kd, v_descale=vd, q_descale=qd)
            elif fp8:
                bq, bk, bv, bkw = q, k8, v8, dict(k_descale=kd, v_descale=vd)
            else:
                bq, bk, bv, bkw = q, kc, vc, {}

        if args.cache_slots:  # B distinct slots of an N-slot pool hold the B-slot cache's rows
            n_slots = args.cache_slots
            idx = torch.randperm(n_slots, generator=torch.Generator().manual_seed(rank))[:b].to(dev)
            idx32 = idx.to(torch.int32)
            raw_k, raw_v = bk.view(torch.uint8), bv.view(torch.uint8)
            pool_k = torch.zeros((n_slots,) + tuple(raw_k.shape[1:]), dtype=torch.uint8, device=dev)
            pool_v = torch.zeros_like(pool_k)
            pool_k[idx], pool_v[idx] = raw_k, raw_v
            pool_k, pool_v = pool_k.view(bk.dtype), pool_v.view(bk.dtype)
            # append Sq new tokens at rows [s - Sq, s) every call (bf16 k / v: quantised into an e4m3 cache)
            kn_app = torch.randn(b, args.sq, args.hkv, d, device=dev, dtype=torch.bfloat16)
            vn_app = torch.randn_like(kn_app)
            sl_app = torch.full((b,), s - args.sq, dtype=torch.int32, device=dev)

            def slot_call():
                return dec.kernel_decode(bq, pool_k, pool_v, sl_app, kn_app, vn_app, True, scale,
                                         cache_batch_idx=idx32, **bkw)

            def slot_plain():
                return dec.kernel_decode(bq, bk, bv, sl_app, kn_app, vn_app, True, scale, **bkw)

            def slot_gather():  # without cache_batch_idx: gather the B slots, a plain call, scatter them back
                gk = pool_k.view(torch.uint8).index_select(0, idx)
                gv = pool_v.view(torch.uint8).index_select(0, idx)
                r = dec.kernel_decode(bq, gk.view(bk.dtype), gv.view(bk.dtype), sl_app, kn_app, vn_app, True, scale,
                                      **bkw)
                pool_k.view(torch.uint8).index_copy_(0, idx, gk)
                pool_v.view(torch.uint8).index_copy_(0, idx, gv)
                return r

        if args.leftpad is not None:  # P pad rows below every sequence's keys, against s - P rows from row 0
            lpad = torch.full((b,), args.leftpad, dtype=torch.int32, device=dev)
            sl_short = torch.full((b,), s - args.leftpad, dtype=torch.int32, device=dev)

            def lp_call():
                return dec.kernel_decode(bq, bk, bv, sl, None, None, True, scale, cache_leftpad=lpad, **bkw)

            def lp_plain():
                return dec.kernel_decode(bq, bk, bv, sl_short, None, None, True, scale, **bkw)

        # SDPA reads the same shard through (B, H, S, D) views
        qt, kt, vt = q.transpose(1, 2), kc.transpose(1, 2), vc.transpose(1, 2)

        def sdpa():
            F.scaled_dot_product_attention(qt, kt, vt, scale=scale, enable_gqa=True)

        rows = {"ours": [], "sdpa": []}
        if args.page_size:
            rows["paged"] = []
        if fp8:
            rows["fp8"] = []
            if args.page_size:
                rows["paged_fp8"] = []
        if q8:
            rows["q8"] = []
            if args.page_size:
                rows["paged_q8"] = []
        mixed_rows = {"mixed_varlen": [], "mixed_padded": [], "mixed_decode_only": []}
        rot_rows = {"rotary_fused": [], "rotary_unfused": [], "rotary_plain": []}
        slot_rows = {"slots": [], "slots_plain": [], "slots_gather_scatter": []}
        lp_rows = {"leftpad": [], "leftpad_plain": []}
        sdpa_err = None
        for _ in range(3):  # alternate them in one run
            rows["ours"].append(time_us(ours, args.iters, args.warmup))
            if args.mixed_chunk:
                mixed_rows["mixed_varlen"].append(time_us(mixed, args.iters, args.warmup))
                mixed_rows["mixed_padded"].append(time_us(padded, args.iters, args.warmup))
                mixed_rows["mixed_decode_only"].append(time_us(decode_only, args.iters, args.warmup))
            if args.rotary:
                rot_rows["rotary_fused"].append(time_us(rot_fused, args.iters, args.warmup))
                rot_rows["rotary_unfused"].append(time_us(rot_unfused, args.iters, args.warmup))
                rot_rows["rotary_plain"].append(time_us(rot_plain, args.iters, args.warmup))
            if args.cache_slots:
                slot_rows["slots"].append(time_us(slot_call, args.iters, args.warmup))
                slot_rows["slots_plain"].append(time_us(slot_plain, args.iters, args.warmup))
                slot_rows["slots_gather_scatter"].append(time_us(slot_gather, args.iters, args.warmup))
            if args.leftpad is not None:
                lp_rows["leftpad"].append(time_us(lp_call, args.iters, args.warmup))
                lp_rows["leftpad_plain"].append(time_us(lp_plain, args.iters, args.warmup))
            if args.page_size:
                rows["paged"].append(time_us(paged, args.iters, args.warmup))
            if fp8:
                rows["fp8"].append(time_us(ours_fp8, args.iters, args.warmup))
                if args.page_size:
                    rows["paged_fp8"].append(time_us(paged_fp8, args.iters, args.warmup))
            if q8:
                rows["q8"].append(time_us(ours_q8, args.iters, args.warmup))
                if args.page_size:
                    rows["paged_q8"].append(time_us(paged_q8, args.iters, args.warmup))
            if sdpa_err is None:
                try:
                    rows["sdpa"].append(time_us(sdpa, args.iters, args.warmup))
                except RuntimeError as e:  # e.g. out of memory when SDPA expands the kv heads
                    sdpa_err = str(e).splitlines()[0][:200]
                    torch.cuda.empty_cache()
        res = dict(cfg, dtype="bf16", world=world, card=name, power_limit=power)
        for k, ts in rows.items():
            if ts:
                us = min(ts)
                nbytes = cfg["fp8_kv_bytes"] if k.endswith(("fp8", "q8")) else cfg["kv_bytes"]
                res[f"{k}_us"] = round(us, 2)
                res[f"{k}_us_all"] = [round(t, 2) for t in ts]
                res[f"{k}_GBps"] = round(nbytes / (us * 1e-6) / 1e9, 1)
                res[f"{k}_share_of_datasheet_hbm"] = round(nbytes / (us * 1e-6) / HBM_DATASHEET_BPS, 3)
        if sdpa_err:
            res["sdpa_error"] = sdpa_err
        if args.mixed_chunk:
            for k, ts in mixed_rows.items():
                res[f"{k}_us"] = round(min(ts), 2)
                res[f"{k}_us_all"] = [round(t, 2) for t in ts]
            res["mixed_speedup_vs_padded"] = round(res["mixed_padded_us"] / res["mixed_varlen_us"], 3)
            # the chunk's rows of the varlen call, bitwise the padded call's (sequence 0 has C tokens in both)
            v_out, p_out = mixed()[0], padded()[0]
            res["mixed_chunk_rows_equal_padded"] = torch.equal(v_out[:c], p_out[0]) if \
                cfg["varlen_splits"] == cfg["padded_splits"] else None
        if args.rotary:
            for k, ts in rot_rows.items():
                res[f"{k}_us"] = round(min(ts), 2)
                res[f"{k}_us_all"] = [round(t, 2) for t in ts]
            res["rotary_fused_over_plain"] = round(res["rotary_fused_us"] / res["rotary_plain_us"], 3)
            res["rotary_speedup_vs_unfused"] = round(res["rotary_unfused_us"] / res["rotary_fused_us"], 3)
            res["rotary_fused_equal_unfused"] = all(torch.equal(x, y) for x, y in zip(rot_fused(), rot_unfused()))
        if args.cache_slots or args.leftpad is not None:
            res["slot_arms_q_dtype"], res["slot_arms_kv_dtype"] = args.q_dtype, args.kv_dtype
        if args.cache_slots:
            for k, ts in slot_rows.items():
                res[f"{k}_us"] = round(min(ts), 2)
                res[f"{k}_us_all"] = [round(t, 2) for t in ts]
            res["slots_over_plain"] = round(res["slots_us"] / res["slots_plain_us"], 3)
            res["slots_speedup_vs_gather_scatter"] = round(res["slots_gather_scatter_us"] / res["slots_us"], 3)
            # every arm appended the same rows to the same contents, so the caches still agree
            res["slots_equal_plain"] = all(torch.equal(x, y) for x, y in zip(slot_call(), slot_plain()))
        if args.leftpad is not None:
            for k, ts in lp_rows.items():
                res[f"{k}_us"] = round(min(ts), 2)
                res[f"{k}_us_all"] = [round(t, 2) for t in ts]
            res["leftpad_over_plain"] = round(res["leftpad_us"] / res["leftpad_plain_us"], 3)
        if args.page_size:
            res["paged_equal_contiguous"] = all(torch.equal(x, y) for x, y in zip(paged(), ours()))
        if fp8:
            res["fp8_speedup_vs_bf16"] = round(res["ours_us"] / res["fp8_us"], 3)
            if args.page_size:
                res["paged_fp8_speedup_vs_paged"] = round(res["paged_us"] / res["paged_fp8_us"], 3)
                res["paged_fp8_equal_contiguous_fp8"] = all(torch.equal(x, y) for x, y in zip(paged_fp8(), ours_fp8()))
            if q8:
                res["q8_speedup_vs_bf16"] = round(res["ours_us"] / res["q8_us"], 3)
                res["q8_speedup_vs_fp8"] = round(res["fp8_us"] / res["q8_us"], 3)
                if args.page_size:
                    res["paged_q8_speedup_vs_paged"] = round(res["paged_us"] / res["paged_q8_us"], 3)
                    res["paged_q8_speedup_vs_paged_fp8"] = round(res["paged_fp8_us"] / res["paged_q8_us"], 3)
                    res["paged_q8_equal_contiguous_q8"] = all(torch.equal(x, y) for x, y in zip(paged_q8(), ours_q8()))
            res.update(fp8_res)
        if world > 1:
            C = dec.cuda_ext.load()
            n_out = b * args.sq * args.hq * d
            mine = torch.randn(n_out + b * args.hq * args.sq, device=dev)
            out = torch.empty(q.shape, dtype=q.dtype, device=dev)
            lse = torch.empty(b, args.hq, args.sq, device=dev)

            def merge():
                C.decode_combine(dec._gather(mine, None, world), out, lse)

            res["allgather_combine_us"] = round(time_us(merge, args.iters, args.warmup), 2)
            res["full_call_us"] = round(time_us(
                lambda: dec.kernel_decode(q, kc, vc, sl, None, None, True, scale, None, world), args.iters,
                args.warmup), 2)
        if rank == 0:
            print(json.dumps(res), flush=True)
        del q, kc, vc
        if args.mixed_chunk:
            del q_pad, q_var, q_one
        if args.rotary:
            del k_new, v_new, cos, sin
        if args.page_size:
            del pk, pv
        if args.cache_slots:
            del pool_k, pool_v, kn_app, vn_app
        if args.cache_slots or args.leftpad is not None:
            del bq, bk, bv, bkw
        if fp8:
            del k8, v8
            if q8:
                del q_e4m3
            if args.page_size:
                del p8k, p8v
        torch.cuda.empty_cache()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
