"""Paged K/V pool on the H100: attention over shuffled pages is bit-equal to the same keys in contiguous rows (decode /
latent-pass kernel and continuation kernel, decoys of tests/test_kv_pages_host.py with NaN in every row a sequence does
not own); System2.generate on a paged pool gives the slotted pool's tokens, latents and K/V rows byte for byte, also
with fragmented pages, evictions and uncached fallbacks; a direct call short of pages is refused with N1_ERR_KV_PAGES
and changes nothing; and the dialog evaluator on a paged pool small enough to evict, and the VLN-CE System-2 evaluator
on one smaller than its largest call, reproduce the runs without a pool and with the slotted pool."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_hopper_kernels_gpu as HK  # noqa: E402
import test_kv_pages_host as KP  # noqa: E402

pytestmark = pytest.mark.gpu
PAGE = 64


def _bits(t):
    return t.view(torch.int16)


def _no_px():
    return torch.empty(0, 1176, dtype=torch.bfloat16, device="cuda")   # a text-only call


# ------------------------------------------------------------------------------------------------ kernels
def _contiguous(d, hkv):
    """The same keys in a slotted layout: sequence b at rows b * cap .. (cap = per * 64), every other row NaN."""
    cap = d["per"] * PAGE
    B = len(d["pairs"])
    k = torch.full((B * cap, hkv * 128), float("nan"), dtype=torch.bfloat16)
    v = k.clone()
    for b, (_, kr, _) in enumerate(d["seqs"]):
        k[b * cap:b * cap + kr.numel()] = d["k"][kr]
        v[b * cap:b * cap + kr.numel()] = d["v"][kr]
    return k.cuda(), v.cuda(), cap


@pytest.mark.parametrize("shuffle", [True, False])
@pytest.mark.parametrize("form", ["decode", "latent"])
def test_decode_attention_over_pages_is_bit_equal_to_contiguous_rows(form, shuffle):
    """attn_kernel (the decode passes and the latent pass): k_len 63 .. 129, GQA 28 / 4."""
    pairs, causal = KP.PAGED_FORMS[form]
    hq, hkv = 28, 4
    d = KP.paged_decoys(pairs, hq, hkv, causal, shuffle=shuffle, seed=3)
    sq, B = pairs[0][0], len(pairs)
    q, k, v = d["q"].cuda(), d["k"].cuda(), d["v"].cuda()
    k_len = torch.tensor([sk for _, sk in pairs], dtype=torch.int32, device="cuda")
    per = d["per"]
    row0 = torch.arange(B, dtype=torch.int32, device="cuda") * per * PAGE
    pages = d["table"].flatten().cuda()
    o = torch.full((B * sq, hq * 128), float("nan"), dtype=torch.bfloat16, device="cuda")
    from internnav_b200 import _lib
    _lib.attention_paged_test(q, k, v, o, hq, hkv, B, sq, k_len, row0, pages, scale=HK.decoy_scale(128))
    kc, vc, cap = _contiguous(d, hkv)
    oc = torch.full_like(o, float("nan"))
    route = _lib.attention_test(q, kc, vc, oc, hq, hkv, 128, B, seq_q=sq, causal=True, scale=HK.decoy_scale(128),
                                k_len=k_len, k_slot=cap)
    torch.cuda.synchronize()
    assert route[0] == "generic"
    assert torch.equal(_bits(o), _bits(oc))
    assert torch.equal(_bits(o.cpu()), _bits(d["expect"]))


@pytest.mark.parametrize("shuffle", [True, False])
def test_continuation_attention_over_pages_is_bit_equal_to_contiguous_rows(shuffle):
    """attn_cache_kernel: chunks after a reused prefix ending on a page boundary (64, 128), a chunk spanning pages
    (keys 50 .. 79), k_len 65 .. 227 with partial last pages, GQA 28 / 4."""
    pairs, causal = KP.PAGED_FORMS["chunk"]
    hq, hkv = 28, 4
    d = KP.paged_decoys(pairs, hq, hkv, causal, shuffle=shuffle, seed=4)
    B, per = len(pairs), d["per"]
    q, k, v = d["q"].cuda(), d["k"].cuda(), d["v"].cuda()
    cu = torch.tensor(np.concatenate([[0], np.cumsum([sq for sq, _ in pairs])]), dtype=torch.int32, device="cuda")
    ctx = torch.tensor([sk - sq for sq, sk in pairs], dtype=torch.int32, device="cuda")
    row0 = torch.arange(B, dtype=torch.int32, device="cuda") * per * PAGE
    from internnav_b200 import _lib
    maxc = max(sq for sq, _ in pairs)
    o = _lib.attention_cache(q, k, v, hq, hkv, cu, ctx, row0, maxc, scale=HK.decoy_scale(128),
                             pages=d["table"].flatten().cuda())
    kc, vc, cap = _contiguous(d, hkv)
    oc = _lib.attention_cache(q, kc, vc, hq, hkv, cu, ctx, row0.clone(), maxc, scale=HK.decoy_scale(128))
    torch.cuda.synchronize()
    assert torch.equal(_bits(o), _bits(oc))
    assert torch.equal(_bits(o.cpu()), _bits(d["expect"]))


# ------------------------------------------------------------------------------------------------ System2.generate
def _setup(seed=5):
    from internnav_b200.qwen import System2
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    s2 = System2(cfg, device="cuda:0")
    s2.load_state_dict(Q.make_s2_state_dict(cfg, seed=seed, lm_head=True))
    return s2


def _px(grids, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(sum(t * h * w for t, h, w in grids), 1176, generator=g).bfloat16().cuda()


def _script(seed):
    """Prompt pieces of _conversation: first turns with their grids and pixels, text-only user turns, look-down turns,
    a fresh prompt, and the look-down frame."""
    from oracle import qwen_oracle as Q
    rng = np.random.Generator(np.random.PCG64(seed))
    g = [[(1, 8, 8), (1, 8, 12)], [(1, 8, 8)], [(1, 12, 8)]]
    gl = (1, 12, 16)
    first = [(Q.make_prompt(rng, 10 + 30 * s, g[s], 6), g[s], _px(g[s], 10 + s)) for s in range(3)]
    text = [Q.make_prompt(rng, 9 + 40 * i, [], 0) for i in range(3)]
    look = [Q.make_prompt(rng, 4, [gl], 3) for _ in range(2)]
    fresh = Q.make_prompt(rng, 70, g[2], 5)
    pxl = _px([gl], 20)
    return first, text, look, fresh, g, gl, pxl


def _conversation(s2, pool, seed=7, between=None):
    """Three rounds on slots 0 .. 2 of `pool`: fresh turns; a text-only dialog continuation (0), a look-down
    continuation (1) and a fresh turn (2) in one batch; two text-only continuations.  `between(round)` runs between the
    rounds.  -> (tokens, latents and reused rows per round, K/V rows per slot)."""
    first, text, look, fresh, g, gl, pxl = _script(seed)
    out = []
    hist = {}
    # round 1: fresh turns
    prompts = [p for p, _, _ in first]
    toks, lat, _ = s2.generate(prompts, torch.cat([x for _, _, x in first]), [gg for _, gs, _ in first for gg in gs],
                               max_new_tokens=5, with_latents=True, past_key_values=[pool.handle(s) for s in range(3)])
    out.append((toks, lat.cpu()))
    caches = s2.last_cache["caches"]
    for s in range(3):
        hist[s] = (prompts[s] + toks[s], list(first[s][1]), [first[s][2]])
    if between:
        between(1)
    # round 2: dialog (0), look-down (1), fresh (2)
    p0 = hist[0][0] + text[0]
    p1 = hist[1][0] + look[0]
    p2 = fresh
    grids = hist[0][1] + hist[1][1] + [gl] + g[2]
    px = torch.cat(hist[0][2] + hist[1][2] + [pxl, first[2][2]])
    toks, lat, _ = s2.generate([p0, p1, p2], px, grids, max_new_tokens=5, with_latents=True,
                               past_key_values=[caches[0], caches[1], caches[2]])
    out.append((toks, lat.cpu(), list(s2.last_cache["reused"])))
    c2 = s2.last_cache["caches"]
    hist[0] = (p0 + toks[0], hist[0][1], hist[0][2])
    hist[1] = (p1 + toks[1], hist[1][1] + [gl], hist[1][2] + [pxl])
    if between:
        between(2)
    # round 3: text-only continuations of 0 and 1
    p0 = hist[0][0] + text[1]
    p1 = hist[1][0] + text[2]
    toks, lat, _ = s2.generate([p0, p1], torch.cat(hist[0][2] + hist[1][2]), hist[0][1] + hist[1][1], max_new_tokens=5,
                               with_latents=True, past_key_values=[c2[0], c2[1]])
    out.append((toks, lat.cpu(), list(s2.last_cache["reused"])))
    rows = {}
    for s in range(3):
        n = pool.valid(s)
        rows[s] = [tuple(x.cpu() for x in pool.read(l, s, 0, n)) for l in range(s2.cfg["layers"])]
    return out, rows


def _same(a, b):
    (oa, ra), (ob, rb) = a, b
    assert len(oa) == len(ob)
    for x, y in zip(oa, ob):
        assert x[0] == y[0]                                   # tokens
        assert torch.equal(_bits(x[1]), _bits(y[1]))          # latents
        assert x[2:] == y[2:]                                 # reused rows
    assert ra.keys() == rb.keys()
    for s in ra:
        assert len(ra[s]) == len(rb[s])
        for (ka, va), (kb, vb) in zip(ra[s], rb[s]):
            assert torch.equal(_bits(ka), _bits(kb)) and torch.equal(_bits(va), _bits(vb))


@pytest.fixture(scope="module")
def s2():
    return _setup()


@pytest.fixture(scope="module")
def slotted(s2):
    from internnav_b200.qwen import KVPool
    return _conversation(s2, KVPool(s2, 5, 1024))


def test_paged_pool_equals_slotted_pool(s2, slotted):
    """Fresh turns, look-down and text-only continuations, mixed batches: byte-identical to the slotted pool."""
    pool = s2.make_paged_kv_pool(5, 64 * 40, 1024)
    got = _conversation(s2, pool)
    _same(got, slotted)
    assert got[0][1][2][0] > 0 and got[0][1][2][1] > 0 and got[0][2][2][0] > 0
    held = sum(pool.slot_pages(s) for s in range(5))
    assert held == sum(-(-pool.valid(s) // PAGE) for s in range(5)) and pool.free_pages + held == 40
    assert pool.bytes == 40 * PAGE * 2 * s2.cfg["layers"] * s2.cfg["kv_heads"] * 128 * 2


def test_fragmented_pages_equal_slotted_pool(s2, slotted):
    """Pages taken and returned by other conversations between the rounds: each conversation's pages end up out of
    order and apart, and the outputs stay byte-identical."""
    from oracle import qwen_oracle as Q
    pool = s2.make_paged_kv_pool(5, 64 * 60, 1024)
    rng = np.random.Generator(np.random.PCG64(99))
    filler = [Q.make_prompt(rng, 150, [], 0) for _ in range(4)]

    def churn(step):   # slot 3 and 4 take pages, 3 gives them back: the next pages taken are scattered
        for s in (3, 4):
            s2.generate([filler[(step + s) % 4]], _no_px(), [], max_new_tokens=3, past_key_values=[pool.handle(s)])
        pool.release(3)
    churn(0)
    got = _conversation(s2, pool, between=churn)
    _same(got, slotted)


def _evicting_run(s2, pool, releases=None):
    """Turns on six conversations (slots 0 .. 5), two at a time, revisiting earlier ones; with `releases` (call index ->
    slots) those slots are released before the call.  -> (outputs, slots released per call by eviction)."""
    from oracle import qwen_oracle as Q
    rng = np.random.Generator(np.random.PCG64(11))
    prompts = {s: Q.make_prompt(rng, 120 + 20 * s, [], 0) for s in range(6)}
    handles = {s: pool.handle(s) for s in range(6)}
    order = [(0, 1), (2, 3), (4, 5), (0, 2), (1, 3), (5, 0), (4, 1)]
    outs, evicted = [], []
    for i, pair in enumerate(order):
        for s in (releases or {}).get(i, ()):
            pool.release(s)
        before = list(pool.version)
        toks, lat, _ = s2.generate([prompts[s] for s in pair], _no_px(), [], max_new_tokens=4, with_latents=True,
                                   past_key_values=[handles[s] for s in pair])
        caches = s2.last_cache["caches"]
        evicted.append([s for s in range(6) if s not in pair and pool.version[s] != before[s]])
        outs.append((toks, lat.cpu(), list(s2.last_cache["reused"])))
        for s, c, t in zip(pair, caches, toks):
            handles[s] = c
            prompts[s] = prompts[s] + t + Q.make_prompt(rng, 15, [], 0)
    rows = {s: [tuple(x.cpu() for x in pool.read(l, s, 0, pool.valid(s))) for l in range(s2.cfg["layers"])]
            for s in range(6) if pool.valid(s) > 0}
    return (outs, rows), evicted


def test_budget_evicts_least_recently_used_and_keeps_outputs(s2):
    """A paged pool for about three of six conversations: calls evict the least recently used conversations outside
    them, and every output and K/V row equals a slotted pool whose same slots are released before the same calls."""
    from internnav_b200.qwen import KVPool
    pool = s2.make_paged_kv_pool(6, 64 * 12, 1024)
    got, evicted = _evicting_run(s2, pool)
    print("evicted per call", evicted, "evictions", pool.evictions)
    assert pool.evictions > 0 and pool.evictions == sum(len(e) for e in evicted)
    # least recently used first: call 2 (slots 4 and 5, 8 pages, 1 free) evicts 0 and 1 (2 + 3 pages, last used in
    # call 0), then 2 (3 pages, call 1)
    assert evicted[:2] == [[], []] and evicted[2] == [0, 1, 2]
    want, _ = _evicting_run(s2, KVPool(s2, 6, 1024), releases={i: e for i, e in enumerate(evicted)})
    _same(got, want)


def test_call_that_cannot_fit_runs_uncached(s2):
    """A call whose pages exceed the whole pool after every other conversation is released runs uncached: no cache is
    returned, the pool is left as it was, and the outputs equal a call without a pool."""
    from oracle import qwen_oracle as Q
    rng = np.random.Generator(np.random.PCG64(12))
    pool = s2.make_paged_kv_pool(4, 64 * 6, 1024)
    small = Q.make_prompt(rng, 90, [], 0)
    s2.generate([small], _no_px(), [], max_new_tokens=4, past_key_values=[pool.handle(3)])
    held, free, valid = pool.slot_pages(3), pool.free_pages, pool.valid(3)
    big = [Q.make_prompt(rng, 200, [], 0) for _ in range(2)]     # 2 x ceil(212 / 64) = 8 pages > 6
    toks, lat, _ = s2.generate(big, _no_px(), [], max_new_tokens=4, with_latents=True,
                               past_key_values=[pool.handle(0), pool.handle(1)])
    assert s2.last_cache["caches"] == [None, None]
    assert (pool.slot_pages(3), pool.free_pages, pool.valid(3)) == (held, free, valid) and pool.evictions == 0
    want, wlat, _ = s2.generate(big, _no_px(), [], max_new_tokens=4, with_latents=True)
    assert toks == want and torch.equal(_bits(lat), _bits(wlat))


def test_direct_generate_short_of_pages_is_refused_and_changes_nothing(s2):
    from internnav_b200 import _lib
    from oracle import qwen_oracle as Q
    rng = np.random.Generator(np.random.PCG64(13))
    pool = s2.make_paged_kv_pool(3, 64 * 5, 1024)
    p0 = Q.make_prompt(rng, 150, [], 0)
    s2.generate([p0], _no_px(), [], max_new_tokens=4, past_key_values=[pool.handle(0)])
    state = (pool.free_pages, [pool.slot_pages(s) for s in range(3)], [pool.valid(s) for s in range(3)])
    rows = [pool.read(l, 0, 0, pool.valid(0)) for l in range(s2.cfg["layers"])]
    p1 = Q.make_prompt(rng, 140, [], 0)                              # ceil(148 / 64) = 3 pages, 2 are free
    L = _lib.lib()
    plan = s2.llm_plan([p1], [], 4, pool, [0], [1])
    nb = L.n1_llm_workspace_bytes(s2._h(), plan)
    ws = s2._scratch("gen", nb)
    eos = (ctypes.c_int32 * 2)(151645, 151643)
    toks, lens, passes = (ctypes.c_int32 * 4)(), (ctypes.c_int32 * 1)(), ctypes.c_int32(0)
    rc = L.n1_llm_generate(s2._h(), plan, _lib.ptr(ws), nb, None, 0, None, 0, eos, 2, 151643, toks, lens, None,
                           ctypes.byref(passes), _lib.stream_ptr())
    msg = L.n1_last_error().decode()
    print(msg)
    assert rc == -8 and "needs 3 pages" in msg and "2 are free" in msg, (rc, msg)
    assert (pool.free_pages, [pool.slot_pages(s) for s in range(3)], [pool.valid(s) for s in range(3)]) == state
    for l in range(s2.cfg["layers"]):
        k, v = pool.read(l, 0, 0, pool.valid(0))
        assert torch.equal(k, rows[l][0]) and torch.equal(v, rows[l][1])


def test_policy_reset_releases_pages():
    import test_dialog_eval_gpu as DT
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from internnav_b200.policy import InternVLAN1Policy
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    m = InternVLAN1ForCausalLM(cfg, device="cuda:0", system1=None)
    m.load_parts(Q.make_s2_state_dict(cfg, seed=3, lm_head=True), None)
    pol = InternVLAN1Policy(m, DT._Processor(), num_envs=2, kv_pool_tokens=64 * 20, system2_only=True)
    caches = pol._caches([0, 1], [False, False], (48, 64))
    assert pol._kv_pool.paged and pol._kv_pool.capacity == pol._kv_capacity(48, 64)
    rng = np.random.Generator(np.random.PCG64(14))
    m._s2.generate([Q.make_prompt(rng, 100, [], 0), Q.make_prompt(rng, 80, [], 0)], _no_px(), [], max_new_tokens=3,
                   past_key_values=caches)
    pool = pol._kv_pool
    assert pool.slot_pages(0) > 0 and pool.slot_pages(1) > 0
    v0 = pool.version[0]
    pol.reset([0])
    assert pool.slot_pages(0) == 0 and pool.valid(0) == 0 and pool.version[0] == v0 + 1 and pool.slot_pages(1) > 0
    assert pool.free_pages == 20 - pool.slot_pages(1)


# ------------------------------------------------------------------------------------------------ closed loops
def _page_budget(record, max_new, nq=4):
    """Pages the largest call of a recorded run needs: a smaller pool runs that call uncached."""
    return max(sum(-(-(n + max_new + nq) // PAGE) for n in lens) for lens in record)


def _evicting_budgets(run, most):
    """Runs on paged pools of `most`, most - 1, ... pages until one evicts -> [(pages, results, evictions)]."""
    tried = []
    for pages in range(most, max(1, most // 3) - 1, -1):
        got, ev = run(pages * PAGE)
        tried.append((pages, got, ev.policy._kv_pool.evictions))
        assert ev.policy._kv_pool.paged
        if tried[-1][2] > 0:
            break
    return tried


def _recording(model, record):
    generate = model.generate

    def gen(prompts, *a, **kw):
        record.append([len(p) for p in prompts])
        return generate(prompts, *a, **kw)
    model.generate = gen


def test_dialog_loop_on_an_evicting_paged_pool(tmp_path):
    import test_dialog_eval_gpu as DT
    from internnav_b200 import habitat_dialog as HD
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    m = InternVLAN1ForCausalLM(cfg, device="cuda:0", system1=None)
    m.load_parts(Q.make_s2_state_dict(cfg, seed=3, lm_head=True), None)
    robots = [0, 1, 2, 3]

    def run(model, kv_pool_tokens=None):
        ev = HD.HabitatDialogEvaluator(model, DT._Processor(), task="instance_dialog", turn=2, num_history=4,
                                       resize_w=112, resize_h=112, max_steps_per_episode=10, max_new_tokens=6,
                                       depth_filter=DT.H.depth_filter, npc=DT._npc, seeds=[40 + r for r in robots],
                                       camera_height=DT.S.CAMERA_HEIGHT, width=DT.SMALL_W, height=DT.SMALL_H,
                                       hfov=DT.S.HFOV, kv_pool_tokens=kv_pool_tokens,
                                       make_follower=lambda env: DT.D.Follower(env._env.sim, 0.25, False))
        logs = {r: [] for r in robots}
        res = ev.run([DT._Env(r, 50 + r, 2, logs[r]) for r in robots])
        return [(rs, logs[r]) for r, rs in zip(robots, res)], ev

    want, _ = run(DT._NoPool(m))
    record = []
    _recording(m, record)
    try:
        slotted, _ = run(m)
    finally:
        del m.generate
    assert slotted == want
    tried = _evicting_budgets(lambda tokens: run(m, tokens), _page_budget(record, 6))
    print("dialog loop: calls", len(record), "(pages, evictions)", [(p, e) for p, _, e in tried])
    assert all(got == want for _, got, _ in tried)
    assert tried[-1][2] > 0


def test_vlnce_system2_loop_on_a_small_paged_pool():
    import test_dialog_eval_gpu as DT
    import test_habitat_eval_s2_gpu as ST
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    m = ST._tiny(None)
    robots = [0, 1, 2, 3]

    def run(model, kv_pool_tokens=None):
        ev = HabitatVLNEvaluator(model, ST._Processor(), mode="system2", num_history=4, resize_w=56, resize_h=56,
                                 max_steps_per_episode=10, max_new_tokens=6, depth_filter=ST.H.depth_filter,
                                 seeds=[40 + r for r in robots], camera_height=ST.S.CAMERA_HEIGHT, width=ST.SMALL_W,
                                 height=ST.SMALL_H, hfov=ST.S.HFOV, kv_pool_tokens=kv_pool_tokens,
                                 make_follower=lambda env: ST.S.ScriptedFollower(env._env.sim, 0.25, False))
        logs = {r: [] for r in robots}
        res = ev.run_system2([ST._Env(r, 50 + r, 2, logs[r]) for r in robots])
        return [(rs, logs[r]) for r, rs in zip(robots, res)], ev

    want, _ = run(DT._NoPool(m))
    record = []
    _recording(m, record)
    try:
        slotted, _ = run(m)
    finally:
        del m.generate
    assert slotted == want
    # This loop calls System 2 for all its environments at once, and an ended episode releases its pages, so no call
    # finds another conversation to evict: a pool smaller than the largest call runs that call uncached instead.
    most = _page_budget(record, 6)
    for pages in (most, most // 2):
        got, ev = run(m, kv_pool_tokens=pages * PAGE)
        print("vln-ce system2 loop: calls", len(record), "pages", pages, "evictions", ev.policy._kv_pool.evictions)
        assert ev.policy._kv_pool.paged and got == want
