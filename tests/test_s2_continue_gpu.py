"""Continuing a System-2 conversation on its K/V cache (the policy's look-down turn), on the GPU: the continued generate
against the fp32 oracle and the library's own full re-prefill.  The chunk attention kernel itself is tested in
tests/test_attention_paths_gpu.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 2e-2
MARGIN = 0.15  # logit units, as tests/test_s2_gpu.py: bf16 near-ties of the greedy pick


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


# ------------------------------------------------------------------------------------------------ two-turn conversation
def _setup(cfg, seed):
    from internnav_b200.qwen import System2
    from oracle import qwen_oracle as Q
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = Q.make_s2_state_dict(cfg, seed=seed, lm_head=True)
    s2 = System2(cfg, device="cuda:0")
    s2.load_state_dict(sd)
    return s2, {k: v.cuda() for k, v in sd.items()}


def _px(grids, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(sum(t * h * w for t, h, w in grids), 1176, generator=g).bfloat16().cuda()


def _two_turns(cfg, seed, grids1, grid_ld, max_new):
    """Turn 1 writes slot 1 of a pool; turn 2 (turn 1 + its answer + a new user turn with the look-down frame) continues
    it.  Checked against the oracle (tokens teacher-forced, latents at the §8d bar) and the library's full re-prefill."""
    from internnav_b200.qwen import KVPool
    from oracle import qwen_oracle as Q
    s2, sd = _setup(cfg, seed)
    rng = np.random.Generator(np.random.PCG64(seed))
    p1 = Q.make_prompt(rng, 12, grids1, 9)
    px1 = _px(grids1, seed)
    pool = KVPool(s2, 3, 2048)
    toks1, _, _ = s2.generate([p1], px1, grids1, max_new_tokens=max_new, with_latents=True,
                              past_key_values=[pool.handle(1)])
    h = s2.last_cache["caches"][0]
    assert h.tokens == p1 + toks1[0] and pool.valid(1) == len(p1) + len(toks1[0])  # TRAJ rows excluded
    p2 = p1 + toks1[0] + Q.make_prompt(rng, 5, [grid_ld], 4)
    grids2 = grids1 + [grid_ld]
    px2 = torch.cat([px1, _px([grid_ld], seed + 1)])
    nh = len(h)
    before = [pool.read(l, 1, 0, nh) for l in range(cfg["layers"])]
    toks2, lat2, _ = s2.generate([p2], px2, grids2, max_new_tokens=max_new, with_latents=True, past_key_values=[h])
    info = s2.last_cache
    assert len(h) == 0  # the call rewrote the slot: the old handle is stale
    assert info["reused"] == [nh] and info["prefill_rows"] == len(p2) - nh
    t, hh, w = grid_ld
    assert info["vit_patches"] == t * hh * w  # only the look-down frame went through the vision tower
    for l in range(cfg["layers"]):  # the reused rows are untouched
        k, v = pool.read(l, 1, 0, nh)
        assert torch.equal(k, before[l][0]) and torch.equal(v, before[l][1])
    # oracle: greedy tokens on the full second-turn prompt, teacher-forced argmax, latents at the §8d bar
    with torch.no_grad():
        ref_toks = Q.greedy_generate(sd, cfg, torch.tensor([p2]), px2.float(), grids2, max_new_tokens=max_new)
        feats = Q.vit_forward(sd, cfg, px2.float(), grids2)
        cur = torch.tensor([p2])
        for tok in toks2[0]:
            lg = Q.next_token_logits(sd, cfg, cur, feats, grids2)
            assert float(lg.max() - lg[tok]) <= MARGIN, (tok, int(lg.argmax()))
            cur = torch.cat([cur, torch.tensor([[tok]])], dim=1)
        ref = Q.generate_latents(sd, cfg, cur, px2.float(), grids2)
        eager = Q.generate_latents({k: v.bfloat16() for k, v in sd.items()}, cfg, cur, px2, grids2)
    print("continued", toks2[0], "oracle", ref_toks)
    assert toks2[0] == ref_toks
    e, ee = _rel(lat2[0], ref[0]), _rel(eager[0], ref[0])
    # the library's own full re-prefill of the same prompt
    toks_f, lat_f, _ = s2.generate([p2], px2, grids2, max_new_tokens=max_new, with_latents=True)
    ef = _rel(lat2, lat_f)
    print("latent rel err vs oracle", e, "bf16 eager", ee, "vs full re-prefill", ef)
    assert e < TOL and e < 2 * ee + 2e-3, (e, ee)
    assert toks_f == toks2 and ef < 1e-2, ef


def test_two_turn_look_down_tiny():
    from oracle import qwen_oracle as Q
    _two_turns(Q.tiny_cfg(), 21, [(1, 8, 8), (1, 8, 12)], (1, 16, 20), 6)


def test_two_turn_look_down_real_width_shallow():
    from oracle import qwen_oracle as Q
    cfg = dict(Q.QWEN25VL_7B)
    cfg.update(v_depth=2, fullatt=[1], layers=2)
    _two_turns(cfg, 22, [(1, 28, 28), (1, 28, 28)], (1, 34, 46), 5)


# ------------------------------------------------------------------------------------------------ batches and the pool
def test_mixed_batch_and_uncached_calls():
    """A batch of a fresh, a continued and a digest-mismatched conversation gives each the tokens of a separate uncached
    call; calls without caches are byte-identical whether or not a pool exists."""
    from internnav_b200.qwen import KVPool
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    s2, _ = _setup(cfg, 31)
    rng = np.random.Generator(np.random.PCG64(31))
    gA, gB, gl = [(1, 8, 8)], [(1, 8, 12)], (1, 12, 16)
    pA, pB = Q.make_prompt(rng, 10, gA, 6), Q.make_prompt(rng, 7, gB, 5)
    pxA, pxB = _px(gA, 1), _px(gB, 2)
    base = s2.generate([pA, pB], torch.cat([pxA, pxB]), gA + gB, max_new_tokens=5, with_latents=True)
    pool = KVPool(s2, 4, 1024)
    t1, lat1, _ = s2.generate([pA, pB], torch.cat([pxA, pxB]), gA + gB, max_new_tokens=5, with_latents=True,
                              past_key_values=[pool.handle(3), pool.handle(0)])
    assert t1 == base[0] and torch.equal(lat1, base[1])  # a fresh pool call is byte-identical to an uncached one
    hA, hB = s2.last_cache["caches"]
    again = s2.generate([pA, pB], torch.cat([pxA, pxB]), gA + gB, max_new_tokens=5, with_latents=True)
    assert again[0] == base[0] and torch.equal(again[1], base[1])  # no cache: untouched by the pool's existence
    # continued (A), digest mismatch (B: same tokens, its image changed), fresh (C)
    pA2 = pA + t1[0] + Q.make_prompt(rng, 4, [gl], 3)
    pB2 = pB + t1[1] + Q.make_prompt(rng, 4, [gl], 3)
    pC = Q.make_prompt(rng, 9, gA, 4)
    pxl, pxB_changed, pxC = _px([gl], 3), _px(gB, 4), _px(gA, 5)
    px = torch.cat([pxA, pxl, pxB_changed, pxl, pxC])
    grids = gA + [gl] + gB + [gl] + gA
    nA = len(hA)
    toks, _, _ = s2.generate([pA2, pB2, pC], px, grids, max_new_tokens=5, with_latents=True,
                             past_key_values=[hA, hB, None])
    info = s2.last_cache
    assert [c.slot for c in info["caches"]] == [3, 0, 1]  # None: a fresh conversation on a never-written slot
    spanB = [i for i, t in enumerate(pB) if t == Q.IMAGE_TOKEN_INDEX][0]
    assert info["reused"] == [nA, spanB, 0], info["reused"]
    for b, (p, pxb, gs) in enumerate([(pA2, torch.cat([pxA, pxl]), gA + [gl]), (pB2, torch.cat([pxB_changed, pxl]), gB + [gl]),
                                      (pC, pxC, gA)]):
        alone, _, _ = s2.generate([p], pxb, gs, max_new_tokens=5, with_latents=True)
        assert toks[b] == alone[0], (b, toks[b], alone[0])


def test_kv_pool_plan_and_generate_errors():
    from internnav_b200 import _lib
    from internnav_b200.qwen import KVPool
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    s2, _ = _setup(cfg, 41)
    pool = KVPool(s2, 2, 64)
    assert pool.bytes == 2 * cfg["layers"] * 2 * 64 * cfg["kv_heads"] * cfg["head_dim"] * 2
    with pytest.raises(_lib.N1Error):
        pool.valid(2)
    L = _lib.lib()
    ids = (__import__("ctypes").c_int32 * 8)(*range(1, 9))
    lens = (__import__("ctypes").c_int32 * 1)(8)
    import ctypes
    p = ctypes.c_void_p()
    for reuse, slot, msg in [(0, 5, b"out of range"), (8, 0, b"reused length"), (0, 0, b"capacity")]:
        new = 60 if msg == b"capacity" else 4
        rc = L.n1_llm_plan_create(s2._h(), ids, lens, 1, (ctypes.c_int32 * 1)(0), 0, new, pool._p,
                                  (ctypes.c_int32 * 1)(reuse), (ctypes.c_int32 * 1)(slot), ctypes.byref(p), _lib.stream_ptr())
        assert rc == -2 and msg in L.n1_last_error(), L.n1_last_error()
    # a reused length beyond what the slot holds is refused at the call
    rc = L.n1_llm_plan_create(s2._h(), ids, lens, 1, (ctypes.c_int32 * 1)(0), 0, 4, pool._p, (ctypes.c_int32 * 1)(3),
                              (ctypes.c_int32 * 1)(0), ctypes.byref(p), _lib.stream_ptr())
    assert rc == 0
    ws = torch.empty(L.n1_llm_workspace_bytes(s2._h(), p), dtype=torch.uint8, device="cuda")
    toks, ln = (ctypes.c_int32 * 4)(), (ctypes.c_int32 * 1)()
    rc = L.n1_llm_generate(s2._h(), p, _lib.ptr(ws), ws.numel(), None, 0, None, 0, None, 0, 0, toks, ln, None, None,
                           _lib.stream_ptr())
    assert rc == -2 and b"holds 0" in L.n1_last_error(), L.n1_last_error()
    L.n1_llm_plan_destroy(p)
