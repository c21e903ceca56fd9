"""Developer microbenchmark of the two tensor-core kernels the benchmark spends its time in, at the benchmark's own shapes
and with the model's own epilogues (bias on qkv and gate/up, residual on o and down): every GEMM tile width (forced
through _lib.gemm_tile) against the dispatcher's choice, and the fused FF block.

    python scripts/bench_tiles.py [--repeats 7] [--out FILE.json]

CUDA events around each launch, the L2 flushed (256 MiB memset) before every timed launch, the variants of one shape
alternated inside the repeat loop so that clock and neighbour drift hits them alike.  Prints the card and its power limit,
then per shape and variant the median time, TFLOP/s at the median and the min-max spread of the repeats, and next to
each forced width the SASS instruction count of the kernel instance it runs (cuobjdump on the built gemm_wgmma.o).
"""
import argparse
import json
import os
import re
import shutil
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from internnav_b200 import _lib  # noqa: E402

ACT_NONE, ACT_SWIGLU = 0, 3
GEMM_SHAPES = [  # (what, M, N, K, act, epilogue operand: "bias" or "residual")
    ("llm gate/up", 19456, 37888, 3584, ACT_SWIGLU, "bias"), ("llm down", 19456, 3584, 18944, ACT_NONE, "residual"),
    ("llm qkv", 19456, 4608, 3584, ACT_NONE, "bias"), ("llm o", 19456, 3584, 3584, ACT_NONE, "residual"),
    ("vit gate/up", 50176, 6848, 1280, ACT_SWIGLU, "bias"), ("vit down", 50176, 1280, 3424, ACT_NONE, "residual"),
    ("vit qkv", 50176, 3840, 1280, ACT_NONE, "bias"), ("vit o", 50176, 1280, 1280, ACT_NONE, "residual"),
]
FF_M = 65536


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def sass_counts():
    """{tile width: SASS instructions of gemm_kernel<BN>}, the instance every row's epilogue runs; {} without cuobjdump"""
    obj = os.path.join(os.path.dirname(_lib.__file__), "_build", "gemm_wgmma.o")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(obj) or not os.path.exists(tool):
        return {}
    r = subprocess.run([tool, "-sass", obj], capture_output=True, text=True)
    counts, bn = {}, None
    for line in r.stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            k = re.search(r"gemm_kernelILi(\d+)EE", m.group(1))
            bn = int(k.group(1)) if k else None
            if bn:
                counts[bn] = 0
        elif bn and re.match(r"\s+/\*[0-9a-f]+\*/\s", line):
            counts[bn] += 1
    return counts


def time_variants(variants, repeats, flush):
    """variants: {name: callable}.  -> {name: [ms, ...]}; one launch of every variant per repeat, in turn."""
    for fn in variants.values():
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in variants}
    for _ in range(repeats):
        for name, fn in variants.items():
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ms[name].append(a.elapsed_time(b))
    return ms


def report(what, flops, ms, rows, sass=None):
    for name, t in ms.items():
        med = statistics.median(t)
        row = dict(shape=what, variant=name, ms=round(med, 4), tflops=round(flops / med / 1e9, 1), min_ms=round(min(t), 4),
                   max_ms=round(max(t), 4))
        n = (sass or {}).get(int(name[2:])) if name.startswith("bn") else None
        if n is not None:
            row["sass"] = n
        rows.append(row)
        print("%-40s %-9s %8.3f ms  %6.1f TFLOP/s  spread %.3f .. %.3f ms%s" % (
            what, name, med, row["tflops"], min(t), max(t), "  %d SASS" % n if n is not None else ""))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_tiles.py needs a GPU"
    name = card()
    print("card: %s (name, power limit, max SM clock)" % name)
    sass = sass_counts()
    print("gemm_kernel<BN> SASS instructions: %s" % (sass or "not available (no cuobjdump or no built object)"))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # > 50 MB L2
    rows = []
    for what, M, N, K, act, operand in GEMM_SHAPES:
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
        n_out = N // 2 if act == ACT_SWIGLU else N
        out = torch.empty(M, n_out, device="cuda", dtype=torch.bfloat16)
        bias = torch.randn(N, device="cuda") if operand == "bias" else None
        res = torch.randn(M, n_out, device="cuda").bfloat16() if operand == "residual" else None
        run = lambda bn: _lib.gemm_tile(x, w, out, bias=bias, residual=res, act=act, tile_n=bn)
        variants = {"auto": lambda: run(0), "bn64": lambda: run(64), "bn128": lambda: run(128), "bn256": lambda: run(256)}
        report("%s %dx%dx%d + %s" % (what, M, N, K, operand), 2.0 * M * N * K, time_variants(variants, args.repeats, flush),
               rows, sass)
        del x, w, out, bias, res
    x = torch.randn(FF_M, 384, device="cuda").bfloat16()
    w1 = (torch.randn(1536, 384, device="cuda") / 384 ** 0.5).bfloat16()
    w2 = (torch.randn(384, 1536, device="cuda") / 1536 ** 0.5).bfloat16()
    b1, b2 = torch.randn(1536, device="cuda"), torch.randn(384, device="cuda")
    lw, lb = torch.randn(384, device="cuda"), torch.randn(384, device="cuda")
    out = torch.empty_like(x)
    variants = {"fused": lambda: _lib.ff_block(x, lw, lb, w1, b1, w2, b2, out=out)}
    report("ff block M=%d" % FF_M, 4.0 * FF_M * 384 * 1536, time_variants(variants, args.repeats, flush), rows)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump({"card": name, "sass": sass, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
