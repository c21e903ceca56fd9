"""Developer microbenchmark of one NavDP decoder layer: each launch of the 9-launch sequence, against the fused
self-attention block, cross-attention block and FF block that replace it (dec_attn_block.cu, ff_block.cu).

    python scripts/bench_dec_layer.py [--repeats 7] [--out FILE.json]

Two sizes: R = 65 536 rows (dual_system: 64 envs x 32 samples x horizon 32) and R = 2 048 (navdp_denoise: 8 x 32 x 8),
34 condition tokens.  CUDA events around each launch, the L2 flushed (256 MiB memset) before every timed launch, the
launches alternated inside the repeat loop (as scripts/bench_tiles.py).  Prints the card and its power limit, then per
launch the median time, its algorithmic TFLOP/s or GB/s, and the min-max spread of the repeats.  Then, per size, both
forms as the sampler runs them: 16 layers with their own weights captured into one CUDA graph, replayed without
flushing the L2, alternated.
"""
import argparse
import json
import math
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_tiles import card, time_variants  # noqa: E402
from internnav_b200 import _lib  # noqa: E402

D, MTOK, LAYERS = 384, 34, 16
SIZES = [("dual_system", 64, 32, 32), ("navdp_denoise", 8, 32, 8)]


def activations(B, Ns, T, gen):
    """Buffers the layers of one pass share; the condition K / V of all 16 layers stacked as the model keeps them."""
    R, dev = B * Ns * T, "cuda"
    x = torch.randn(R, D, generator=gen).bfloat16().to(dev)
    return dict(x=x, ln=torch.empty_like(x), q=torch.empty_like(x),
                qkv=torch.empty(R, 3 * D, dtype=torch.bfloat16, device=dev),
                ckv=torch.randn(B * MTOK, LAYERS * 2 * D, generator=gen).bfloat16().to(dev))


def layer(B, Ns, T, gen, acts, l=0):
    """Weights of decoder layer l at this size, and the launches of both forms.  -> (sequence, fused): lists of
    (name, callable, flops, bytes moved)."""
    R = B * Ns * T
    dev = "cuda"
    w = lambda n, k: (torch.randn(n, k, generator=gen) / math.sqrt(k)).bfloat16().to(dev)
    v = lambda n, s=0.1: (torch.randn(n, generator=gen) * s).to(dev)
    wqkv, bqkv, wo1, bo1 = w(3 * D, D), v(3 * D), w(D, D), v(D)
    wq, bq, wo2, bo2 = w(D, D), v(D), w(D, D), v(D)
    w1, b1, w2, b2 = w(1536, D), v(1536), w(D, 1536), v(D)
    lns = [(1 + v(D), v(D)) for _ in range(3)]
    x, ln, qkv, q = acts["x"], acts["ln"], acts["qkv"], acts["q"]
    ckv = acts["ckv"][:, l * 2 * D:(l + 1) * 2 * D]
    bf = 2  # bytes per element
    act = R * D * bf
    seq = [
        ("qkv gemm", lambda: _lib.gemm(ln, wqkv, bias=bqkv, out=qkv), 2.0 * R * 3 * D * D, act + 3 * act),
        ("self attention", lambda: _lib.attention(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], 8, 8, 48, B * Ns, T, T,
                                                  causal=True), 4.0 * R * T * D, 4 * act),
        ("sa_out gemm + residual", lambda: _lib.gemm(q, wo1, bias=bo1, residual=x, out=x), 2.0 * R * D * D, 3 * act),
        ("layernorm (norm2)", lambda: _lib.layernorm(x, *lns[1], out=ln), 0.0, 2 * act),
        ("ca_q gemm", lambda: _lib.gemm(ln, wq, bias=bq, out=q), 2.0 * R * D * D, 2 * act),
        ("cross attention", lambda: _lib.attention(q, ckv[:, :D], ckv[:, D:], 8, 8, 48, B * Ns, T, MTOK, kv_div=Ns),
         4.0 * R * MTOK * D, 2 * act),
        ("ca_out gemm + residual", lambda: _lib.gemm(q, wo2, bias=bo2, residual=x, out=x), 2.0 * R * D * D, 3 * act),
        ("ff block", lambda: _lib.ff_block(x, *lns[2], w1, b1, w2, b2, out=x), 4.0 * R * D * 1536, 2 * act),
        ("layernorm (next norm1)", lambda: _lib.layernorm(x, *lns[0], out=ln), 0.0, 2 * act),
    ]
    fused = [
        ("sa block", lambda: _lib.dec_sa_block(x, *lns[0], wqkv, bqkv, wo1, bo1, B, Ns, T),
         2.0 * R * 4 * D * D + 4.0 * R * T * D, 2 * act),
        ("ca block", lambda: _lib.dec_ca_block(x, *lns[1], wq, bq, wo2, bo2, ckv, MTOK, B, Ns, T),
         2.0 * R * 2 * D * D + 4.0 * R * MTOK * D, 2 * act),
        ("ff block", lambda: _lib.ff_block(x, *lns[2], w1, b1, w2, b2, out=x), 4.0 * R * D * 1536, 2 * act),
    ]
    return seq, fused


def graph_of(fns):
    """One CUDA graph that issues the launches `fns` in order (warmed up once first)."""
    for fn in fns:
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for fn in fns:
            fn()
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dec_layer.py needs a GPU"
    name = card()
    print("card: %s (name, power limit, max SM clock)" % name)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    for what, B, Ns, T in SIZES:
        gen = torch.Generator().manual_seed(0)
        acts = activations(B, Ns, T, gen)
        seq, fused = layer(B, Ns, T, gen, acts)
        R = B * Ns * T
        variants = {("seq", n): fn for n, fn, _, _ in seq}
        variants.update({("fused", n): fn for n, fn, _, _ in fused if n != "ff block"})
        ms = time_variants(variants, args.repeats, flush)
        print("\n%s: R = %d (B %d x Ns %d x T %d), %d condition tokens" % (what, R, B, Ns, T, MTOK))
        totals = {"seq": 0.0, "fused": 0.0}
        for form, launches in (("seq", seq), ("fused", fused)):
            for n, _, flops, nbytes in launches:
                t = ms[("seq", n)] if n == "ff block" else ms[(form, n)]
                med = statistics.median(t)
                totals[form] += med
                row = dict(size=what, R=R, form=form, launch=n, ms=round(med, 4), min_ms=round(min(t), 4),
                           max_ms=round(max(t), 4), tflops=round(flops / med / 1e9, 1), gbps=round(nbytes / med / 1e6, 1))
                rows.append(row)
                print("  %-5s %-24s %8.4f ms  %6.1f TFLOP/s  %7.1f GB/s  spread %.4f .. %.4f" % (
                    form, n, med, row["tflops"], row["gbps"], min(t), max(t)))
        print("  layer total: 9-launch sequence %.3f ms, fused (3 launches) %.3f ms" % (totals["seq"], totals["fused"]))
        rows.append(dict(size=what, R=R, seq_total_ms=round(totals["seq"], 4), fused_total_ms=round(totals["fused"], 4)))
        # As the sampler runs them: 16 layers with their own weights (together ~66 MB, more than the L2) back to back from
        # one CUDA graph, the L2 not flushed.
        stack = [(seq, fused)] + [layer(B, Ns, T, gen, acts, l) for l in range(1, LAYERS)]
        graphs = {form: graph_of([fn for pair in stack for _, fn, _, _ in pair[i]])
                  for i, form in enumerate(("seq", "fused"))}
        no_flush = torch.empty(1, dtype=torch.uint8, device="cuda")
        ms = time_variants({k: g.replay for k, g in graphs.items()}, args.repeats, no_flush)
        for form in ("seq", "fused"):
            t = ms[form]
            med = statistics.median(t)
            print("  16 layers, own weights, one graph, no flush: %-5s %8.4f ms  spread %.4f .. %.4f" % (form, med, min(t),
                                                                                                     max(t)))
            rows.append(dict(size=what, R=R, form=form, launch="16 layers, own weights, graph, no flush", ms=round(med, 4),
                             min_ms=round(min(t), 4), max_ms=round(max(t), 4)))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump({"card": name, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
