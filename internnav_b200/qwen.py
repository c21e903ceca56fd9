"""Host-side driver of the System-2 path (Qwen2.5-VL vision tower + decoder prefill) over libn1b200.so.

`System2` owns the packed weights (inside the library handle) and caches integer plans; its methods are the batched
equivalents of the calls InternVLAN1ForCausalLM.generate_latents makes (internvla_n1.py L320-347):
`visual(pixel_values, grid_thw)` and `model(inputs_embeds, position_ids)` + the last-n_query slice.
"""
import ctypes
import itertools
from collections import OrderedDict

import numpy as np
import torch

from . import _lib
from ._lib import S2Dims, TensorDesc, c_void_p, check

QWEN25VL_7B = dict(
    v_depth=32, v_hidden=1280, v_heads=16, v_inter=3420, v_patch=14, v_tpatch=2, v_merge=2, v_window=112, v_out=3584,
    fullatt=[7, 15, 23, 31],
    layers=28, hidden=3584, heads=28, kv_heads=4, head_dim=128, inter=18944, vocab=152064,
    rms_eps=1e-6, rope_theta=1000000.0, mrope=[16, 24, 24], n_query=4)


def _dims_struct(cfg):
    d = S2Dims()
    for k in ("v_depth", "v_hidden", "v_heads", "v_inter", "v_patch", "v_tpatch", "v_merge", "v_window", "v_out",
              "layers", "hidden", "heads", "kv_heads", "head_dim", "inter", "vocab", "n_query"):
        setattr(d, k, int(cfg[k]))
    d.n_fullatt = len(cfg["fullatt"])
    for i, v in enumerate(cfg["fullatt"]):
        d.fullatt[i] = int(v)
    d.rms_eps, d.rope_theta = float(cfg["rms_eps"]), float(cfg["rope_theta"])
    for i in range(3):
        d.mrope[i] = int(cfg["mrope"][i])
    return d


EOS_TOKEN_IDS = (151645, 151643)  # Qwen2.5-VL generation_config.json: <|im_end|>, <|endoftext|>
PAD_TOKEN_ID = 151643


def normalise_keys(state_dict):
    """Accept the transformers 4.51 layout (`visual.*`, `model.*`) and the 5.x one (`model.visual.*`,
    `model.language_model.*`); System-1 keys (`model.navdp.*`) are dropped, `lm_head.weight` is kept for generate()."""
    out = {}
    for k, v in state_dict.items():
        if k.startswith("model.visual."):
            k = k[len("model."):]
        elif k.startswith("model.language_model."):
            k = "model." + k[len("model.language_model."):]
        if k.startswith("model.navdp."):
            continue
        if k.startswith("visual.") or k.startswith("model.") or k == "lm_head.weight":
            out[k] = v
    return out


IMAGE_TOKEN_ID = 151655


def _i32(a):
    """ctypes int32 pointer into a C-contiguous int32 numpy array (the array must outlive the call)."""
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))


def image_spans(prompt, grids, merge=2):
    """(first token, token count) of every image of a prompt, in order; `grids` are the prompt's image grids."""
    spans, i, k = [], 0, 0
    while i < len(prompt):
        if prompt[i] == IMAGE_TOKEN_ID:
            t, h, w = (int(v) for v in grids[k])
            n = t * h * w // (merge * merge)
            spans.append((i, n))
            i, k = i + n, k + 1
        else:
            i += 1
    return spans


def reuse_length(handle_tokens, handle_images, prompt, images, cap, need):
    """Rows of a cached conversation a new prompt may reuse: the longest common token prefix, cut
      * at the first image of the prompt whose content digest differs from the cached one at the same position (every
        image token has the same id, so only the digest tells two images apart),
      * at the first image the prefix would split,
      * below the prompt length (the last prompt row must be prefilled: its logits start the decode).
    handle_tokens: ids the cache holds K/V for; handle_images / images: {first token: (count, digest)} and [(first token,
    count, digest)].  0 when the conversation does not fit the slot (`need` rows > `cap`)."""
    if need > cap:
        return 0
    n = 0
    m = min(len(handle_tokens), len(prompt) - 1)
    while n < m and handle_tokens[n] == prompt[n]:
        n += 1
    for st, cnt, dg in images:
        if st >= n:
            break
        if st + cnt > n or handle_images.get(st) != (cnt, dg):
            return st
    return n


class KVCache:
    """One conversation's K/V in a slot of a KVPool (HF's `past_key_values` for one prompt): the token ids it covers and
    the position, length and content digest of each image among them.  A handle is stale once its slot is rewritten."""

    def __init__(self, pool, slot, tokens=(), images=None, version=None):
        self.pool, self.slot = pool, int(slot)
        self.tokens = list(tokens)
        self.images = dict(images or {})
        self.version = pool.version[self.slot] if version is None else version

    def __len__(self):
        return len(self.tokens) if self.version == self.pool.version[self.slot] else 0


PAGE_TOKENS = 64  # tokens per page of a paged KVPool


def _pages(tokens):
    return -(-int(tokens) // PAGE_TOKENS)


class KVPool:
    """Caller-owned device memory for `slots` conversations of up to `capacity` tokens, sized once.

    With `pages` the pool is paged: `pages` pages of 64 tokens shared by all slots, `capacity` the most one conversation
    may hold.  A slot holds pages only for the tokens its conversation has, so the pool can be much smaller than slots x
    capacity; generate() evicts the least recently used conversations when a call needs more pages than are free."""
    _serials = itertools.count()

    def __init__(self, s2, slots, capacity, pages=None):
        L = _lib.lib()
        self.s2, self.slots, self.capacity = s2, int(slots), int(capacity)
        self.pages = None if pages is None else int(pages)
        h = c_void_p()
        with torch.cuda.device(s2.device):
            if self.pages is None:
                check(L.n1_kv_pool_create(s2._h(), self.slots, self.capacity, ctypes.byref(h)))
            else:
                check(L.n1_kv_pool_create_paged(s2._h(), self.slots, self.pages, self.capacity, ctypes.byref(h)))
        self._p = h
        self.serial = next(KVPool._serials)  # identifies the pool in System2's plan cache (ids and addresses are reused)
        self.version = [0] * self.slots
        self.last_use = {}  # slot -> number of the generate() call that last used it (paged pools: eviction order)
        self.evictions = 0  # conversations generate() released to make room

    @property
    def paged(self):
        return self.pages is not None

    @property
    def bytes(self):
        return int(_lib.lib().n1_kv_pool_bytes(self._p))

    @property
    def free_pages(self):
        return int(_lib.lib().n1_kv_pool_free_pages(self._p))

    def slot_pages(self, slot):
        r = _lib.lib().n1_kv_pool_slot_pages(self._p, int(slot))
        if r < 0:
            check(r)
        return r

    def release(self, slot):
        """End the conversation of `slot`: its handles go stale and a paged pool gets its pages back."""
        check(_lib.lib().n1_kv_pool_release(self._p, int(slot)))
        self.version[int(slot)] += 1
        self.last_use.pop(int(slot), None)

    def make_room(self, slots, keep_rows, need_rows):
        """Pages for one call on a paged pool: sequence b on slots[b] keeps keep_rows[b] rows and needs need_rows[b].
        Releases the least recently used conversations outside the call until the free pages cover the call.  -> False
        (nothing released) when even releasing every other conversation would not."""
        need = sum(_pages(n) - _pages(k) for k, n in zip(keep_rows, need_rows))
        short = need - self.free_pages - sum(self.slot_pages(s) - _pages(k) for s, k in zip(slots, keep_rows))
        if short <= 0:
            return True
        inside = set(slots)
        others = sorted((s for s in range(self.slots) if s not in inside and self.slot_pages(s) > 0),
                        key=lambda s: (self.last_use.get(s, -1), s))
        if sum(self.slot_pages(s) for s in others) < short:
            return False
        for s in others:
            if short <= 0:
                break
            short -= self.slot_pages(s)
            self.release(s)
            self.evictions += 1
        return True

    def valid(self, slot):
        r = _lib.lib().n1_kv_pool_valid(self._p, int(slot))
        if r < 0:
            check(r)
        return r

    def read(self, layer, slot, row, n):
        """(K, V) rows [row, row + n) of `slot` in decoder layer `layer`: bf16 [n, kv_heads * head_dim] copies."""
        w = self.s2.cfg["kv_heads"] * self.s2.cfg["head_dim"]
        k = torch.empty(n, w, device=self.s2.device, dtype=torch.bfloat16)
        v = torch.empty_like(k)
        check(_lib.lib().n1_kv_pool_read(self._p, int(layer), int(slot), int(row), int(n), _lib.ptr(k), _lib.ptr(v),
                                         _lib.stream_ptr()))
        return k, v

    def handle(self, slot):
        """An empty cache on `slot`: passing it to generate() writes the conversation there."""
        return KVCache(self, slot)

    def __del__(self):
        try:
            if self._p:
                _lib.lib().n1_kv_pool_destroy(self._p)
        except Exception:
            pass


class ImageFeaturePool:
    """Caller-owned device memory for vision-tower output kept across calls: bf16 [rows, v_out], sized once (7 168 B per
    row at the 7B shapes; a 392 x 392 frame is 196 rows, a 640 x 480 one 391).  An entry holds the merged rows of one
    image, keyed by (content digest, t, h, w).  Rows are taken from a free list one at a time, so an entry's rows need
    not be adjacent and freed rows serve any image.  A call that needs rows evicts the least recently used entries it
    does not itself use."""

    def __init__(self, s2, rows):
        if int(rows) <= 0:
            raise ValueError("ImageFeaturePool: rows must be positive")
        self.rows = int(rows)
        self.feats = torch.empty(self.rows, s2.cfg["v_out"], device=s2.device, dtype=torch.bfloat16)
        self._free = list(range(self.rows - 1, -1, -1))  # popped from the end: lowest row first
        self._entries = OrderedDict()                    # key -> int32 rows, least recently used first

    @property
    def bytes(self):
        return self.feats.numel() * self.feats.element_size()

    @property
    def free_rows(self):
        return len(self._free)

    def __len__(self):
        return len(self._entries)

    def __contains__(self, key):
        return key in self._entries

    def keys(self):
        """Entry keys, least recently used first."""
        return list(self._entries)

    def rows_of(self, key):
        return self._entries[key].tolist()

    def assign(self, keys, counts):
        """Rows for the images of one call: image i has key keys[i] and counts[i] merged rows.  Entries that exist become
        the most recently used; every other distinct key gets rows from the free list, after evicting least recently
        used entries outside this call as needed.  -> (rows of each image, set of keys that got new rows: the caller
        fills those, or discards them if it cannot).  ValueError when the call's distinct images need more rows than
        the pool has."""
        need = OrderedDict()
        for k, n in zip(keys, counts):
            need[k] = int(n)
        total = sum(need.values())
        if total > self.rows:
            raise ValueError("ImageFeaturePool: one call needs %d rows of image features, the pool has %d" % (total, self.rows))
        for k in need:
            if k in self._entries:
                self._entries.move_to_end(k)
        new = [k for k in need if k not in self._entries]
        want = sum(need[k] for k in new)
        while len(self._free) < want:  # entries this call uses are at the end, so the oldest is never one of them
            _, rows = self._entries.popitem(last=False)
            self._free.extend(rows[::-1].tolist())
        for k in new:
            self._entries[k] = np.array([self._free.pop() for _ in range(need[k])], dtype=np.int32)
        return [self._entries[k] for k in keys], set(new)

    def discard(self, keys):
        """Drop entries (rows whose features were never written) and return their rows to the free list."""
        for k in keys:
            rows = self._entries.pop(k, None)
            if rows is not None:
                self._free.extend(rows[::-1].tolist())


class System2:
    def __init__(self, cfg=None, device="cuda:0"):
        self.cfg = dict(QWEN25VL_7B if cfg is None else cfg)
        self.device = torch.device(device)
        self._handle = None
        self._vit_plans, self._llm_plans = {}, {}
        self._ws = {}
        self._calls = 0

    def make_paged_kv_pool(self, slots, tokens, max_tokens_per_slot=None):
        """A paged KVPool of ceil(tokens / 64) pages for `slots` conversations of at most `max_tokens_per_slot` tokens
        (default: the whole pool)."""
        pages = _pages(tokens)
        return KVPool(self, slots, pages * PAGE_TOKENS if max_tokens_per_slot is None else max_tokens_per_slot, pages)

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, state_dict):
        L = _lib.lib()
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError("n1b200 has no CPU path: System2 needs device='cuda:N'")
        sd = normalise_keys(state_dict)
        h = c_void_p()
        check(L.n1_create(ctypes.byref(h), dev.index or 0))
        keep, descs = [], []
        for name, t in sd.items():
            if t.dtype not in (torch.float32, torch.bfloat16):
                t = t.float()
            t = t.detach().to(dev).contiguous()
            keep.append(t)
            d = TensorDesc()
            d.name, d.data, d.dtype = name.encode(), t.data_ptr(), _lib.dtype_code(t)
            d.ndim = 1
            d.shape[0] = t.numel()
            descs.append(d)
        arr = (TensorDesc * len(descs))(*descs)
        dims = _dims_struct(self.cfg)
        with torch.cuda.device(dev):
            check(L.n1_s2_load(h, ctypes.byref(dims), arr, len(descs), _lib.stream_ptr()))
            torch.cuda.synchronize()
        self._handle = h
        del keep

    def __del__(self):
        try:
            L = _lib.lib()
            for p in self._vit_plans.values():
                L.n1_vit_plan_destroy(p)
            for p in self._llm_plans.values():
                L.n1_llm_plan_destroy(p)
            if self._handle is not None:
                L.n1_destroy(self._handle)
        except Exception:
            pass

    @property
    def has_latent_queries(self):
        """Whether the loaded state_dict held `model.latent_queries` (a System-2-only checkpoint has none)."""
        return bool(_lib.lib().n1_s2_has_latent_queries(self._h()))

    def _h(self):
        if self._handle is None:
            raise RuntimeError("System-2 weights not loaded")
        return self._handle

    def _scratch(self, key, nbytes):
        k = (key, torch.cuda.current_stream().cuda_stream)
        buf = self._ws.get(k)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=self.device)
            self._ws[k] = buf
        return buf

    # ------------------------------------------------------------------ plans (integer host work, cached by shape)
    def vit_plan(self, grid_thw):
        key = tuple(int(v) for g in grid_thw for v in g)
        p = self._vit_plans.get(key)
        if p is None:
            L = _lib.lib()
            arr = (ctypes.c_int32 * len(key))(*key)
            p = c_void_p()
            with torch.cuda.device(self.device):
                check(L.n1_vit_plan_create(self._h(), arr, len(key) // 3, ctypes.byref(p), _lib.stream_ptr()))
            self._vit_plans[key] = p
        return p

    def llm_plan(self, prompts, grid_thw, max_new_tokens=0, pool=None, reused=None, slots=None):
        """Decoder plan, cached by its arguments.  prompts: list of token-id lists (no TRAJ tokens); grid_thw: image grids
        in prompt order across the batch.  max_new_tokens 0: a latent plan (prefill_latents); >= 1: a generation plan,
        which with a KVPool `pool` continues sequence b on slot slots[b], whose first reused[b] tokens it reuses."""
        gkey = tuple(int(v) for g in grid_thw for v in g)
        cont = None if pool is None else (pool.serial, tuple(reused), tuple(slots))
        key = (int(max_new_tokens), tuple(tuple(p) for p in prompts), gkey, cont)
        p = self._llm_plans.get(key)
        if p is None:
            L = _lib.lib()
            B = len(prompts)
            flat = [int(t) for q in prompts for t in q]
            ids = (ctypes.c_int32 * len(flat))(*flat)
            lens = (ctypes.c_int32 * B)(*[len(q) for q in prompts])
            garr = (ctypes.c_int32 * max(1, len(gkey)))(*gkey)
            per_seq = lambda v: None if pool is None else (ctypes.c_int32 * B)(*v)
            p = c_void_p()
            with torch.cuda.device(self.device):
                check(L.n1_llm_plan_create(self._h(), ids, lens, B, garr, len(gkey) // 3, int(max_new_tokens),
                                           None if pool is None else pool._p, per_seq(reused), per_seq(slots),
                                           ctypes.byref(p), _lib.stream_ptr()))
            self._evict_plans(L)
            self._llm_plans[key] = p
        return p

    def _evict_plans(self, L, keep=8):
        """Prompts change every step in deployment, so the cache only serves repeated calls within a step (generate +
        latents).  Oldest first: the library recycles a destroyed plan's device block, and the oldest plan's consumers
        finished long ago, so the recycling never has to wait."""
        while len(self._llm_plans) > keep:
            k = next(iter(self._llm_plans))
            L.n1_llm_plan_destroy(self._llm_plans.pop(k))

    def positions(self, plan, B):
        L = _lib.lib()
        n = L.n1_llm_plan_tokens(plan)
        pos = (ctypes.c_int32 * (3 * n))()
        dl = (ctypes.c_int32 * B)()
        check(L.n1_llm_plan_positions(plan, pos, dl))
        return torch.tensor(list(pos), dtype=torch.int64).view(3, n), torch.tensor(list(dl), dtype=torch.int64)

    # ------------------------------------------------------------------ hot calls
    def visual(self, pixel_values, grid_thw, feature_pool=None, dst_rows=None):
        """self.visual(pixel_values, grid_thw=image_grid_thw): [N, 1176] -> [N/4, hidden] bf16.  With an ImageFeaturePool
        merged row r goes to feature_pool.feats[dst_rows[r]] instead (int32, no row twice) and nothing is returned."""
        L = _lib.lib()
        plan = self.vit_plan(grid_thw)
        px = pixel_values.to(self.device, torch.bfloat16).contiguous()
        n = L.n1_vit_plan_patches(plan)
        assert px.shape[0] == n, "pixel_values rows (%d) do not match image_grid_thw (%d patches)" % (px.shape[0], n)
        if feature_pool is None:
            out, dst = torch.empty(n // (self.cfg["v_merge"] ** 2), self.cfg["v_out"], device=self.device,
                                   dtype=torch.bfloat16), None
        else:
            out, dst = feature_pool.feats, np.ascontiguousarray(dst_rows, dtype=np.int32)
        nb = L.n1_vit_workspace_bytes(self._h(), plan)
        ws = self._scratch("vit", nb)
        check(L.n1_qwen_vit(self._h(), plan, _lib.ptr(ws), nb, _lib.ptr(px), _lib.ptr(out), out.shape[0],
                            None if dst is None else _i32(dst), 0 if dst is None else len(dst), _lib.stream_ptr()))
        return out if feature_pool is None else None

    def _pool_features(self, feature_pool, px, grid_thw, digests, images):
        """Image features of grid_thw[i] for i in `images` (in plan order) through `feature_pool`: the images it does not
        hold go through the vision tower in one call, into freshly taken rows.  -> (int32 row table of the plan's image
        tokens, patches encoded).  Sets self.last_features."""
        merge2 = self.cfg["v_merge"] ** 2
        sizes = [int(t) * int(h) * int(w) for t, h, w in grid_thw]
        start = np.concatenate([[0], np.cumsum(sizes)]).tolist()
        keys = [(int(digests[i]),) + tuple(int(v) for v in grid_thw[i]) for i in images]
        rows, new = feature_pool.assign(keys, [sizes[i] // merge2 for i in images])
        miss, seen = [], set()
        for i, k, r in zip(images, keys, rows):
            if k in new and k not in seen:
                seen.add(k)
                miss.append((i, r))
        hits = sum(1 for k in keys if k not in new)
        if miss:
            try:
                sub = torch.cat([px[start[i]:start[i + 1]] for i, _ in miss]) if len(miss) < len(grid_thw) else px
                self.visual(sub, [grid_thw[i] for i, _ in miss], feature_pool, np.concatenate([r for _, r in miss]))
            except Exception:
                feature_pool.discard(new)
                raise
        patches = sum(sizes[i] for i, _ in miss)
        self.last_features = dict(image_hits=hits, vit_patches=patches)
        table = np.concatenate(rows) if rows else np.zeros(0, dtype=np.int32)
        return table, patches

    def prefill_latents(self, prompts, image_feats, grid_thw):
        """Embedding splice + decoder prefill + last-n_query slice for B prompts -> [B, n_query, hidden] bf16."""
        L = _lib.lib()
        plan = self.llm_plan(prompts, grid_thw)
        B = len(prompts)
        feats = image_feats.to(self.device, torch.bfloat16).contiguous()
        assert feats.shape[0] == L.n1_llm_plan_image_tokens(plan), "image features and image tokens do not match"
        out = torch.empty(B, self.cfg["n_query"], self.cfg["hidden"], device=self.device, dtype=torch.bfloat16)
        nb = L.n1_llm_workspace_bytes(self._h(), plan)
        ws = self._scratch("llm", nb)
        check(L.n1_llm_prefill(self._h(), plan, _lib.ptr(ws), nb, _lib.ptr(feats), _lib.ptr(out), _lib.stream_ptr()))
        return out

    def generate_latents(self, prompts, pixel_values, grid_thw):
        """Batched InternVLAN1ForCausalLM.generate_latents: one prompt per environment, images in prompt order."""
        return self.prefill_latents(prompts, self.visual(pixel_values, grid_thw), grid_thw)

    # ------------------------------------------------------------------ training branch (UNVALIDATED on GPU, see s2_train.cu)
    def train_forward(self, prompts, pixel_values, grid_thw, image_feats=None):
        """Hidden states at the TRAJ positions for a training batch (prompts WITHOUT the TRAJ tokens): [B, n_query, H].
        Keeps the K/V cache and the per-layer TRAJ-row tensors for `train_backward` (same prompts, next call)."""
        L = _lib.lib()
        plan = self.llm_plan(prompts, grid_thw, 1)
        feats = self.visual(pixel_values, grid_thw) if image_feats is None else image_feats
        feats = feats.to(self.device, torch.bfloat16).contiguous()
        out = torch.empty(len(prompts), self.cfg["n_query"], self.cfg["hidden"], device=self.device, dtype=torch.bfloat16)
        nb = L.n1_s2_train_workspace_bytes(self._h(), plan)
        ws = self._scratch("train", nb)
        check(L.n1_s2_train_forward(self._h(), plan, _lib.ptr(ws), nb, _lib.ptr(feats), _lib.ptr(out), _lib.stream_ptr()))
        self._train_state = (plan, ws, nb)
        return out

    def set_latent_queries(self, latent_queries):
        """Push updated `latent_queries` ([1, n_query, H] or [n_query, H]) into the library after an optimizer step."""
        t = latent_queries.reshape(self.cfg["n_query"], self.cfg["hidden"]).to(self.device, torch.bfloat16).contiguous()
        check(_lib.lib().n1_s2_set_latent_queries(self._h(), _lib.ptr(t), _lib.stream_ptr()))
        torch.cuda.current_stream().synchronize()

    def train_backward(self, grad_states):
        """d loss / d traj states [B, n_query, H] -> d loss / d latent_queries fp32 [1, n_query, H]."""
        plan, ws, nb = self._train_state
        g = grad_states.to(self.device, torch.bfloat16).contiguous()
        out = torch.empty(1, self.cfg["n_query"], self.cfg["hidden"], device=self.device, dtype=torch.float32)
        check(_lib.lib().n1_s2_train_backward(self._h(), plan, _lib.ptr(ws), nb, _lib.ptr(g), _lib.ptr(out),
                                              _lib.stream_ptr()))
        return out

    def generate(self, prompts, pixel_values, grid_thw, max_new_tokens=128, eos_token_ids=EOS_TOKEN_IDS,
                 pad_token_id=PAD_TOKEN_ID, with_latents=False, image_feats=None, past_key_values=None, feature_pool=None):
        """Greedy decode for B prompts (`model.generate(do_sample=False, max_new_tokens=...)`, internvla_n1_policy.py
        L169-176).  Returns (list of B generated-token lists, each ending with its eos id unless the budget ran out,
        latents [B, n_query, hidden] or None, decode passes run).  With `with_latents` the K/V cache of the decode is
        extended by the TRAJ tokens, which equals `generate_latents(output_ids, ...)` without a second prefill.
        `image_feats`: the vision tower's output for every image, used instead of `pixel_values`.
        `past_key_values`: one entry per prompt, a KVCache of one KVPool (an empty one for a fresh prompt; all slots
        distinct) or None: a fresh conversation on a slot no other entry uses (one never written if there is one, else the
        lowest; a cache held elsewhere on that slot goes stale).  Prompt b reuses reuse_length(...) rows of its slot: only
        the images after that prefix go through the vision tower and only the rows after it are prefilled.  Afterwards the
        slot holds the new conversation and `self.last_cache` = dict(caches=[one new KVCache per prompt], prefill_rows,
        vit_patches, reused).  A batch in which some conversation does not fit its slot runs as an uncached call and
        returns None for every cache.  On a paged pool the call first takes the pages it needs, releasing the least
        recently used conversations outside the call (their handles go stale, so their next turn prefills in full); when
        even that does not make room, the call runs uncached.
        `feature_pool`: an ImageFeaturePool; images it holds skip the vision tower, the others are encoded into it, and
        `self.last_features` = dict(image_hits, vit_patches).  The outputs are byte-identical to a call without it."""
        if image_feats is not None and (feature_pool is not None or past_key_values is not None):
            raise ValueError("generate: image_feats excludes feature_pool and past_key_values")
        B, nq = len(prompts), self.cfg["n_query"]
        caches = pool = None
        if past_key_values is not None:
            if len(past_key_values) != B or all(c is None for c in past_key_values):
                raise ValueError("past_key_values: one KVCache or None per prompt, at least one KVCache")
            given = [c for c in past_key_values if c is not None]
            pool = given[0].pool
            if any(c.pool is not pool for c in given) or len({c.slot for c in given}) != len(given):
                raise ValueError("past_key_values: the caches of one call must be distinct slots of one KVPool")
            # a None entry starts a fresh conversation on a slot no other entry uses: one never written first, then the lowest
            free = sorted((s_ for s_ in range(pool.slots) if s_ not in {c.slot for c in given}),
                          key=lambda s_: (pool.valid(s_) > 0, s_))
            if len(free) < B - len(given):
                raise ValueError("past_key_values: the pool has no free slot for a None entry")
            free = iter(free)
            caches = [c if c is not None else pool.handle(next(free)) for c in past_key_values]
            if any(len(p) + int(max_new_tokens) + nq > pool.capacity for p in prompts):
                pool = None   # some conversation does not fit its slot: an uncached call
        L = _lib.lib()
        if not L.n1_s2_has_lm_head(self._h()):
            raise RuntimeError("generate() needs lm_head.weight in the loaded state_dict; there is no fallback")
        px = None if image_feats is not None else pixel_values.to(self.device, torch.bfloat16).contiguous()
        digests = self.image_digests(px, grid_thw) if pool is not None or feature_pool is not None else None
        # the rows each prompt reuses, and the images after that prefix: only those need features
        reused, keep, images = [0] * B, list(range(len(grid_thw))), []
        if pool is not None:
            keep, gi = [], 0
            for b, (p, c) in enumerate(zip(prompts, caches)):
                spans = image_spans(p, grid_thw[gi:], self.cfg["v_merge"])
                imgs = [(st, n, digests[gi + k]) for k, (st, n) in enumerate(spans)]
                r = reuse_length(c.tokens, c.images, p, imgs, pool.capacity, len(p) + int(max_new_tokens) + nq) \
                    if len(c) else 0
                reused[b] = min(r, pool.valid(c.slot)) if r else 0
                keep += [gi + k for k, (st, _, _) in enumerate(imgs) if st >= reused[b]]
                images.append({st: (n, dg) for st, n, dg in imgs})
                gi += len(spans)
            need = [len(p) + int(max_new_tokens) + nq for p in prompts]
            if pool.paged and not pool.make_room([c.slot for c in caches], reused, need):
                pool, reused, keep = None, [0] * B, list(range(len(grid_thw)))   # no room even after eviction: uncached
        sizes = [int(t) * int(h) * int(w) for t, h, w in grid_thw]
        feats, table = image_feats, None
        if feature_pool is not None:
            table, vit_patches = self._pool_features(feature_pool, px, grid_thw, digests, keep)
            feats = feature_pool.feats
        else:
            vit_patches = sum(sizes[i] for i in keep)
            if feats is None and keep:
                start = np.cumsum([0] + sizes).tolist()
                sub = px if len(keep) == len(grid_thw) else torch.cat([px[start[i]:start[i + 1]] for i in keep])
                feats = self.visual(sub, [grid_thw[i] for i in keep])
        if feats is not None:
            feats = feats.to(self.device, torch.bfloat16).contiguous()
        slots = None if pool is None else [c.slot for c in caches]
        plan = self.llm_plan(prompts, grid_thw, max_new_tokens, pool, reused, slots)
        lat = torch.empty(B, nq, self.cfg["hidden"], device=self.device, dtype=torch.bfloat16) if with_latents else None
        nb = L.n1_llm_workspace_bytes(self._h(), plan)
        ws = self._scratch("gen", nb)
        eos = (ctypes.c_int32 * max(1, len(eos_token_ids)))(*[int(e) for e in eos_token_ids])
        toks = (ctypes.c_int32 * (B * int(max_new_tokens)))()
        lens = (ctypes.c_int32 * B)()
        passes = ctypes.c_int32(0)
        for s_ in slots or ():   # the call rewrites these slots: every older handle on them is stale from here on
            pool.version[s_] += 1
        check(L.n1_llm_generate(self._h(), plan, _lib.ptr(ws), nb, _lib.ptr(feats), 0 if feats is None else feats.shape[0],
                                None if table is None else _i32(table), 0 if table is None else len(table), eos,
                                len(eos_token_ids), int(pad_token_id), toks, lens, _lib.ptr(lat), ctypes.byref(passes),
                                _lib.stream_ptr()))
        out = [list(toks[b * max_new_tokens: b * max_new_tokens + lens[b]]) for b in range(B)]
        self._calls += 1
        for s_ in slots or ():
            pool.last_use[s_] = self._calls
        if caches is not None:
            new = [None] * B if pool is None else \
                [KVCache(pool, s_, (p + o)[:pool.valid(s_)], im) for p, o, s_, im in zip(prompts, out, slots, images)]
            self.last_cache = dict(caches=new, prefill_rows=int(L.n1_llm_plan_tokens(plan)), vit_patches=vit_patches,
                                   reused=reused)
        return out, lat, passes.value

    def image_digests(self, px, grid_thw):
        """Content digest (uint64 as int64) of every image of device bf16 pixel rows `px`, computed on the device."""
        sizes = [int(t) * int(h) * int(w) for t, h, w in grid_thw]
        off = torch.tensor([0] + sizes, dtype=torch.int64).cumsum(0).to(self.device)
        out = torch.empty(len(sizes), dtype=torch.int64, device=self.device)
        check(_lib.lib().n1_image_digest(_lib.ptr(px), px.shape[1], _lib.ptr(off), len(sizes), _lib.ptr(out),
                                         _lib.stream_ptr()))
        return out.tolist()
