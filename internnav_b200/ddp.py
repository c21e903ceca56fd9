"""Data-parallel gradient exchange of the training step (SURVEY.md §8e, row a13): one process per GPU, the trainable
tensors (System-1 parameters minus the detached RGB ViT, plus `latent_queries`) all-reduced once per step in buckets.

The reference trains through HF Trainer -> torch DistributedDataParallel with `ddp_bucket_cap_mb=100`
(scripts/train/base_train/train.py L249).  What is reproduced here is DDP's observable contract:

  * bucket layout: parameters walked in order, a first bucket of 1 MiB then buckets of `bucket_cap_mb`, split by
    dtype, launched in reverse order because backward produces gradients last-parameter-first
    (`torch.distributed._compute_bucket_assignment_by_size` + the reversal in DistributedDataParallel.__init__) --
    pinned against that very function in tests/test_ddp_gloo.py;
  * arithmetic: every local gradient is divided by the world size, then summed across ranks.

What is different by construction: gradients LIVE in the bucket buffers (`GradientBuckets.grads` are views), so a
backward kernel writes its result where the collective reads it and nothing is copied or re-flattened per step; each
bucket is one `all_reduce` on the caller's process group (NCCL over NVLink/NVSwitch on H100s, gloo in the CPU tests),
issued asynchronously so that the remaining backward overlaps it.
"""
from collections import OrderedDict

import torch
import torch.distributed as dist

FIRST_BUCKET_BYTES = 1024 * 1024  # torch.distributed._DEFAULT_FIRST_BUCKET_BYTES


def bucket_assignment(named_shapes, bucket_cap_mb=100, first_bucket_bytes=FIRST_BUCKET_BYTES):
    """named_shapes: ordered {name: (shape, dtype)} in parameter order -> list of buckets (lists of names) in LAUNCH
    order (the bucket holding the last parameters first)."""
    cap = int(bucket_cap_mb * 1024 * 1024)
    limits = [first_bucket_bytes, cap]
    open_buckets = {}   # dtype -> [names, bytes, limit index]
    done = []
    for name, (shape, dtype) in named_shapes.items():
        n = 1
        for s in shape:
            n *= int(s)
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        b = open_buckets.setdefault(dtype, [[], 0, 0])
        b[0].append(name)
        b[1] += nbytes
        if b[1] >= limits[min(b[2], len(limits) - 1)]:
            done.append((min_index(b[0], named_shapes), b[0]))
            open_buckets[dtype] = [[], 0, b[2] + 1]
    for b in open_buckets.values():
        if b[0]:
            done.append((min_index(b[0], named_shapes), b[0]))
    done.sort(key=lambda t: t[0])       # torch sorts buckets by their smallest parameter index ...
    return [names for _, names in reversed(done)]   # ... and DDP launches them in reverse


def min_index(names, named_shapes):
    order = {n: i for i, n in enumerate(named_shapes)}
    return min(order[n] for n in names)


class GradientBuckets:
    def __init__(self, named_shapes, device, bucket_cap_mb=100, process_group=None):
        self.named_shapes = OrderedDict(named_shapes)
        self.group = process_group
        self.layout = bucket_assignment(self.named_shapes, bucket_cap_mb)
        self.buffers, self.grads = [], OrderedDict()
        for names in self.layout:
            dtype = self.named_shapes[names[0]][1]
            sizes = [int(torch.Size(self.named_shapes[n][0]).numel()) for n in names]
            buf = torch.zeros(sum(sizes), dtype=dtype, device=device)
            off = 0
            for n, sz in zip(names, sizes):
                self.grads[n] = buf[off:off + sz].view(self.named_shapes[n][0])
                off += sz
            self.buffers.append(buf)
        self._pending = []

    def zero(self):
        for b in self.buffers:
            b.zero_()

    def bucket_of(self, name):
        """Index (launch order) of the bucket holding `name`."""
        for i, names in enumerate(self.layout):
            if name in names:
                return i
        raise KeyError(name)

    def scale_(self, factor, skip=()):
        for i, b in enumerate(self.buffers):
            if i not in skip:
                b.mul_(factor)

    def all_reduce(self, async_op=True, skip=(), only=None, append=False):
        """Average buckets over the process group, last parameters first.  `skip` / `only` select buckets by index, so a
        caller can exchange the buckets that are complete while the rest of the backward still runs (what DDP's hooks do)
        and the remaining ones afterwards (`append=True` keeps the earlier handles pending).  With async_op the
        collectives are in flight on return (call wait() before the optimizer reads the gradients)."""
        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError("GradientBuckets.all_reduce needs an initialised torch.distributed process group")
        world = dist.get_world_size(self.group)
        if not append:
            self._pending = []
        for i, buf in enumerate(self.buffers):
            if i in skip or (only is not None and i not in only):
                continue
            buf.div_(world)
            work = dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.group, async_op=async_op)
            if async_op:
                self._pending.append(work)
        return self

    def wait(self):
        for w in self._pending:
            w.wait()
        self._pending = []


def trainable_shapes(navdp_shapes, latent_query_shape, dtype=torch.float32):
    """The tensors the reference's training step updates, in parameter order: every System-1 tensor except the RGB
    ViT, whose tokens are detached (navdp_backbone.py L170-171; see tests/golden/s1_training_reference.npz), followed by
    `latent_queries`."""
    out = OrderedDict()
    for name, shape in navdp_shapes.items():
        if name.startswith("rgbd_encoder.rgb_model."):
            continue
        out["model.navdp." + name] = (tuple(shape), dtype)
    out["model.latent_queries"] = (tuple(latent_query_shape), dtype)
    return out
