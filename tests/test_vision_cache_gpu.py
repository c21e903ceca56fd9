"""The System-2 vision-feature pool on the GPU.  The vision tower treats each image on its own, so an image's features
are the same bytes in any batch; the pool rests on that.  Calls with a pool, with or without the K/V pool and through
the policy, give byte-identical tokens, latents and actions to calls without one, and encode only the images the pool
does not hold."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from vl_processor import qwen_processor  # noqa: E402

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int16).cpu()


def _px(grids, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(sum(t * h * w for t, h, w in grids), 1176, generator=g).bfloat16().cuda()


def test_vision_features_are_batch_invariant():
    """Mixed sizes at the 7B vision widths: each image's features alone, in batches of other orders and compositions,
    in a 64-image batch, and written through a row map into a pool are the same bytes."""
    from internnav_b200.qwen import ImageFeaturePool, System2
    from oracle import qwen_oracle as Q
    cfg = dict(Q.QWEN25VL_7B)
    cfg.update(v_depth=4, fullatt=[1, 3], layers=1)
    s2 = System2(cfg, device="cuda:0")
    s2.load_state_dict(Q.make_s2_state_dict(cfg, seed=3, device="cuda", dtype=torch.bfloat16, vocab_rows=256))
    grids = [(1, 28, 28), (1, 34, 46), (1, 16, 16), (1, 10, 14), (1, 6, 22), (1, 22, 6), (1, 2, 2), (1, 18, 30)]
    pxs = [_px([g], 100 + i) for i, g in enumerate(grids)]
    alone = [_bits(s2.visual(p, [g])) for p, g in zip(pxs, grids)]
    merged = [t * h * w // 4 for t, h, w in grids]

    def check(order):
        out = _bits(s2.visual(torch.cat([pxs[i] for i in order]), [grids[i] for i in order]))
        r = 0
        for i in order:
            assert torch.equal(out[r:r + merged[i]], alone[i]), (order, i)
            r += merged[i]

    check(list(range(len(grids))))
    check(list(reversed(range(len(grids)))))
    check([3, 0, 5])
    check([1, 1, 2, 7, 0])
    check([i % len(grids) for i in range(64)])
    # through a row map: scattered rows of a pool, nothing else written
    pool = ImageFeaturePool(s2, 4096)
    pool.feats.fill_(7.0)
    order = [4, 0, 2]
    dst = np.random.default_rng(0).permutation(4096)[:sum(merged[i] for i in order)].astype(np.int32)
    s2.visual(torch.cat([pxs[i] for i in order]), [grids[i] for i in order], pool, dst)
    got = _bits(pool.feats)
    r = 0
    for i in order:
        assert torch.equal(got[torch.from_numpy(dst[r:r + merged[i]]).long()], alone[i]), i
        r += merged[i]
    untouched = np.setdiff1d(np.arange(4096), dst)
    assert torch.equal(got[torch.from_numpy(untouched).long()], _bits(torch.full((len(untouched), cfg["v_out"]), 7.0).bfloat16()))


def _model(seed):
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from internnav_b200.manifest import random_navdp_state_dict
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    model = InternVLAN1ForCausalLM(cfg, device="cuda:0")
    model.load_parts(Q.make_s2_state_dict(cfg, seed=seed, lm_head=True), random_navdp_state_dict(seed=seed + 1,
                                                                                                    vlm_token_dim=cfg["hidden"]))
    return model


def _episode(seed):
    """Three calls over images a..g of mixed sizes for two environments: fresh turns that share images with earlier
    calls, then look-down turns continuing the second call.  -> list of calls (prompts, per-prompt image ids)."""
    from oracle import qwen_oracle as Q
    rng = np.random.Generator(np.random.PCG64(seed))
    img = {k: g for k, g in zip("abcdefgL", [(1, 8, 8), (1, 8, 12), (1, 12, 8), (1, 6, 10), (1, 8, 8), (1, 10, 6),
                                            (1, 8, 8), (1, 12, 16)])}
    px = {k: _px([g], 1000 * seed + i) for i, (k, g) in enumerate(img.items())}
    fresh = [["abc", "de"], ["acf", "dg"]]
    calls = []
    for imgs in fresh:
        calls.append(([Q.make_prompt(rng, 7, [img[k] for k in s], 5) for s in imgs], imgs))
    return img, px, calls, rng


def _run(model, seed, kv, features, max_new=5):
    """The episode of _episode(seed); with `kv` the look-down turns continue on a K/V pool, with `features` every call
    goes through that feature pool.  -> per call (generated, latent bytes, vit_patches, image_hits)."""
    from oracle import qwen_oracle as Q
    img, px, calls, rng = _episode(seed)
    kvpool = model.make_kv_pool(2, 1024) if kv else None
    out, last = [], None

    def call(prompts, imgs, caches):
        grids = [img[k] for s in imgs for k in s]
        pixels = torch.cat([px[k] for s in imgs for k in s])
        kw = {}
        if caches is not None:
            kw["past_key_values"] = caches
        if features is not None:
            kw["feature_pool"] = features
        o = model.generate_with_latents(prompts, pixels, grids, max_new_tokens=max_new, **kw)
        out.append((o.generated, _bits(o.latents), getattr(o, "vit_patches", None), getattr(o, "image_hits", None)))
        return o

    for prompts, imgs in calls:
        last = call(prompts, imgs, [kvpool.handle(0), kvpool.handle(1)] if kv else None)
        last_prompts, last_imgs = prompts, imgs
    # look-down turns: previous prompt + answer + a user turn with frame L
    p2 = [p + g + Q.make_prompt(rng, 4, [img["L"]], 3) for p, g in zip(last_prompts, last.generated)]
    call(p2, [s + "L" for s in last_imgs], last.past_key_values if kv else None)
    return out, img


@pytest.mark.parametrize("kv", [False, True], ids=["no_kv", "kv_pool"])
def test_pool_outputs_identical_and_encode_misses_only(kv):
    model = _model(11)
    base, img = _run(model, 5, kv, None)
    pool = model.make_feature_pool(4096)
    got, _ = _run(model, 5, kv, pool)
    seen = set()
    for c, ((tb, lb, _, _), (tg, lg, patches, hits)) in enumerate(zip(base, got)):
        assert tg == tb and torch.equal(lg, lb), c
        # the images this call needs: all of them, or on a continued look-down turn only the new frame
        need = ["L", "L"] if (kv and c == 2) else [k for s in (["abc", "de"], ["acf", "dg"], ["acfL", "dgL"])[c] for k in s]
        miss = [k for k in dict.fromkeys(need) if k not in seen]
        assert patches == sum(img[k][1] * img[k][2] for k in miss), (c, patches, miss)
        assert hits == sum(1 for k in need if k in seen), (c, hits)
        seen.update(need)
    assert got[1][3] == 3   # images a, c and d come from the pool


def test_small_pool_evicts_and_outputs_stay_identical():
    model = _model(13)
    base, img = _run(model, 6, True, None)
    pool = model.make_feature_pool(100)   # the first call needs 95 rows, the episode's images 174
    got, _ = _run(model, 6, True, pool)
    for (tb, lb, _, _), (tg, lg, _, _) in zip(base, got):
        assert tg == tb and torch.equal(lg, lb)
    total = sum(img[k][1] * img[k][2] // 4 for k in "abcdefgL")
    assert pool.rows < total and len(pool) < len(img)
    with pytest.raises(ValueError, match="rows of image features"):
        _run(model, 6, False, model.make_feature_pool(40))


def test_row_table_and_feature_count_checks():
    """The entry points refuse a row table of the wrong length or with a row outside the pool, and without a row table
    features of the wrong length, before anything runs."""
    import ctypes
    from internnav_b200 import _lib
    from internnav_b200.qwen import ImageFeaturePool, _i32
    model = _model(17)
    s2 = model._s2
    L = _lib.lib()
    grids = [(1, 8, 8)]
    plan = s2.vit_plan(grids)
    pool = ImageFeaturePool(s2, 32)
    px = _px(grids, 1)
    nb = L.n1_vit_workspace_bytes(s2._h(), plan)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")

    def vit(rows):
        a = np.asarray(rows, dtype=np.int32)
        return L.n1_qwen_vit(s2._h(), plan, _lib.ptr(ws), nb, _lib.ptr(px), _lib.ptr(pool.feats), pool.rows, _i32(a),
                             len(a), _lib.stream_ptr()), L.n1_last_error().decode()

    assert vit(range(16))[0] == 0
    assert vit(range(15))[0] == -2 and "16" in vit(range(15))[1]
    rc, msg = vit(list(range(15)) + [32])
    assert rc == -2 and "outside the pool" in msg
    rc, msg = vit([0] * 16)
    assert rc == -2 and "twice" in msg
    rc = L.n1_qwen_vit(s2._h(), plan, _lib.ptr(ws), nb, _lib.ptr(px), _lib.ptr(pool.feats), pool.rows, None, 0,
                       _lib.stream_ptr())   # without a table the output has exactly the 16 merged rows
    assert rc == -2 and "16" in L.n1_last_error().decode(), L.n1_last_error()
    from oracle import qwen_oracle as Q
    prompt = Q.make_prompt(np.random.Generator(np.random.PCG64(1)), 3, grids, 2)
    gp = s2.llm_plan([prompt], grids, 2)
    gnb = L.n1_llm_workspace_bytes(s2._h(), gp)
    gws = torch.empty(gnb, dtype=torch.uint8, device="cuda")
    toks, lens = (ctypes.c_int32 * 2)(), (ctypes.c_int32 * 1)()
    for rows, msg in [(range(15), "entries"), (list(range(15)) + [-1], "outside the pool")]:
        a = np.asarray(rows, dtype=np.int32)
        rc = L.n1_llm_generate(s2._h(), gp, _lib.ptr(gws), gnb, _lib.ptr(pool.feats), pool.rows, _i32(a), len(a), None, 0,
                               0, toks, lens, None, None, _lib.stream_ptr())
        assert rc == -2 and msg in L.n1_last_error().decode(), L.n1_last_error()
    rc = L.n1_llm_generate(s2._h(), gp, _lib.ptr(gws), gnb, _lib.ptr(pool.feats), 15, None, 0, None, 0, 0, toks, lens, None,
                           None, _lib.stream_ptr())   # without a table the features have exactly the 16 image-token rows
    assert rc == -2 and "16" in L.n1_last_error().decode(), L.n1_last_error()


def _raw(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, (*shape, 3), dtype=np.uint8)


class _Recorder:
    """Forwards the model; records each generate_with_latents call's prompts, ids, latents and vision patches."""

    def __init__(self, model):
        self.m, self.config, self.device, self.calls = model, model.config, model.device, []

    def make_kv_pool(self, slots, capacity):
        return self.m.make_kv_pool(slots, capacity)

    def make_feature_pool(self, rows):
        self.pool = self.m.make_feature_pool(rows)
        return self.pool

    def generate_with_latents(self, prompts, pixels, grids, **kw):
        out = self.m.generate_with_latents(prompts, pixels, grids, **kw)
        patches = out.vit_patches if "feature_pool" in kw else \
            int(sum(int(t) * int(h) * int(w) for t, h, w in torch.as_tensor(grids).tolist()))
        self.calls.append(dict(prompts=prompts, generated=out.generated, latents=_bits(out.latents), patches=patches))
        return out


def test_policy_episode_with_vision_cache():
    """A scripted episode (fresh turns with history, look-down turns, mixed calls) gives the same prompts, ids, latents
    and actions with and without the vision cache, and the cache encodes fewer patches."""
    from internnav_b200.policy import InternVLAN1Policy
    model = _model(21)
    proc = qwen_processor()
    off, on = _Recorder(model), _Recorder(model)
    kw = dict(num_envs=3, num_history=4, resize_w=100, resize_h=90, max_new_tokens=6)
    p_off, p_on = InternVLAN1Policy(off, proc, **kw), InternVLAN1Policy(on, proc, vision_cache_frames=4, **kw)
    assert p_off._vl is not None and p_off._feature_pool is None

    def frame(k, e):
        return _raw((96, 128), 100 * k + e)

    results = []
    for k in range(9):
        for pol in (p_off, p_on):
            pol.step_no_infer([0, 1, 2], [frame(k, e) for e in range(3)])
        if k % 2 == 1:
            for env_ids, look in (([0, 1, 2], [False] * 3), ([2, 0], [True, False])):
                res = [pol.s2_step(env_ids, [frame(50 + k, e) for e in env_ids], None, None,
                                   ["go to door %d" % e for e in env_ids], None, look) for pol in (p_off, p_on)]
                for r in res:
                    assert all(not isinstance(x, Exception) for x in r), r
                results.append(res)
    assert on.pool is p_on._feature_pool and p_on._feature_pool is not None
    assert len(off.calls) == len(on.calls) == 8
    for a, b in zip(off.calls, on.calls):
        assert a["prompts"] == b["prompts"] and a["generated"] == b["generated"]
        assert torch.equal(a["latents"], b["latents"])
    for r_off, r_on in results:
        for x, y in zip(r_off, r_on):
            assert x.output_action == y.output_action
            assert (x.output_pixel is None) == (y.output_pixel is None)
            if x.output_latent is not None:
                assert torch.equal(_bits(x.output_latent), _bits(y.output_latent))
    n_off, n_on = sum(c["patches"] for c in off.calls), sum(c["patches"] for c in on.calls)
    print("ViT patches without / with the vision cache:", n_off, n_on)
    assert n_on < n_off
