"""System-2 image inputs per call: the host path (Pillow + the PIL-backed Qwen2-VL image processor) against the device
path (QwenImagePreprocessor).

    python scripts/bench_s2_inputs.py [--batches 8,64] [--repeats 7] [--out FILE]

Two turns per environment, as InternVLAN1Policy prepares them:
  * fresh: the new 480 x 640 raw frame is resized to 384 x 384 and joins 8 history frames (already 384 x 384); all 9
    images are processed (384^2 -> 392^2, 784 rows each);
  * look-down: the same 9 images plus the 480 x 640 frame at full size (-> 476 x 644).
Host path: Pillow resize of the new frame (fresh turn), the image processor on every prompt image of each environment,
torch.cat, and the copy to a device bf16 tensor.  Device path: one upload of the raw frames, their resize, and
QwenImagePreprocessor over every image of the call (history frames already on the device).  Both end in a device
synchronise; they run alternated, `--repeats` times each, and the rows of the two paths are checked bit-equal.  The
card's name and power limit and the host CPU model and core count are read in the same run.
"""
import argparse
import json
import os
import platform
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def host_cpu():
    """CPU model (lscpu, else /proc/cpuinfo, else the machine type) and the logical core count."""
    try:
        out = subprocess.run(["lscpu"], capture_output=True, text=True).stdout
    except OSError:
        out = ""
    try:
        with open("/proc/cpuinfo") as fh:
            out += fh.read()
    except OSError:
        pass
    names = [ln.split(":", 1)[1].strip() for ln in out.splitlines() if ln.lower().startswith(("model name", "model name:"))]
    return "%s, %d cores" % (names[0] if names else platform.machine(), os.cpu_count() or 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="8,64")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_s2_inputs needs a GPU"
    from transformers.models.qwen2_vl.image_processing_pil_qwen2_vl import Qwen2VLImageProcessorPil
    from internnav_b200.preprocess import QwenImagePreprocessor
    ip = Qwen2VLImageProcessorPil(min_pixels=3136, max_pixels=12845056)
    vl = QwenImagePreprocessor.from_hf(ip, "cuda:0")
    assert vl is not None
    lines = [{"card": card(), "host_cpu": host_cpu(), "torch_threads": torch.get_num_threads()}]
    print(json.dumps(lines[0]), flush=True)
    for B in [int(b) for b in a.batches.split(",")]:
        rng = np.random.default_rng(B)
        raw = rng.integers(0, 256, (B, 480, 640, 3), dtype=np.uint8)            # this call's frames
        hist_pil = [[Image.fromarray(rng.integers(0, 256, (384, 384, 3), dtype=np.uint8)) for _ in range(8)]
                    for _ in range(B)]
        hist_dev = [[torch.from_numpy(np.array(im)).cuda() for im in h] for h in hist_pil]
        new_pil = [Image.fromarray(raw[b]).resize((384, 384)) for b in range(B)]
        new_dev = vl.resize(raw, (384, 384))

        def host(turn):
            if turn == "fresh":
                imgs = [h + [Image.fromarray(raw[b]).resize((384, 384))] for b, h in enumerate(hist_pil)]
            else:
                imgs = [h + [new_pil[b], Image.fromarray(raw[b])] for b, h in enumerate(hist_pil)]
            px = torch.cat([ip(images=im, return_tensors="pt")["pixel_values"] for im in imgs])
            return px.to("cuda", torch.bfloat16)

        def device(turn):
            x = torch.from_numpy(raw).cuda()
            if turn == "fresh":
                x = vl.resize(x, (384, 384))
                imgs = [im for b, h in enumerate(hist_dev) for im in h + [x[b]]]
            else:
                imgs = [im for b, h in enumerate(hist_dev) for im in h + [new_dev[b], x[b]]]
            return vl(imgs)[0]

        for turn in ("fresh", "look_down"):
            assert torch.equal(host(turn), device(turn)), (B, turn)   # also the warm-up of both paths
            times = {"host": [], "device": []}
            for _ in range(a.repeats):
                for name, fn in (("host", host), ("device", device)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    rows = fn(turn)
                    torch.cuda.synchronize()
                    times[name].append((time.perf_counter() - t0) * 1e3)
            line = {"B": B, "turn": turn, "rows": rows.shape[0], "bit_equal": True}
            for name, t in times.items():
                line[name + "_ms"] = {"median": round(statistics.median(t), 3), "min": round(min(t), 3),
                                      "max": round(max(t), 3)}
            line["speedup"] = round(line["host_ms"]["median"] / line["device_ms"]["median"], 1)
            lines.append(line)
            print(json.dumps(line), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
