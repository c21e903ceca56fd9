"""The decoy construction and checks of tests/test_attention_paths_gpu.py on the CPU: at every head dim and in the
offset (chunk / decode) form the target beats every visible key by more than 20 nats and the float64 reference rounds
exactly to the expected V; and the exact check and the float64 bound both reject references that carry the errors
those tests exist to catch (a causal offset one key off, k_len +- 1, row0 one row off, kv_div reading the next
environment, the last partial 64-key block dropped, the GQA head map h % Hkv, a continuation attending with ctx = 0)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_hopper_kernels_gpu as H  # noqa: E402

SCALE = 0.0625


def _pool(pairs, hd, hq, hkv, causal, mode, share=1, seed=0, nan_rest=False):
    """Query sequence b = (sq, sk) reads K/V sequence kb = b // share, which lives in slot nkv - kb of a pool whose
    slots hold cap rows of key code (decoys) or random data, so reads past k_len or before row0 see real keys; with
    nan_rest, every row but the sequences' keys is NaN instead, as in the GPU tests' pools.
    -> (q, k, v, seqs = [(q_rows, k_rows, vis)], expect or None, k0 per query sequence, cap)."""
    gen = torch.Generator().manual_seed(seed)
    nkv = (len(pairs) + share - 1) // share
    cap = max(sk for _, sk in pairs) + 64
    slots = nkv + 1
    rows_q = sum(sq for sq, _ in pairs)
    q = torch.zeros(rows_q, hq * hd)
    k = torch.zeros(slots * cap, hkv * hd)
    v = H.decoy_values(slots * cap, hkv * hd, gen) if mode == "decoy" else torch.randn(slots * cap, hkv * hd, generator=gen)
    for s in range(slots):
        if mode == "decoy":
            k[s * cap:(s + 1) * cap] = H.decoy_key_code(cap, 1, hd).repeat(1, hkv)
        else:
            kk = torch.randn(cap, hkv, hd, generator=gen) * 1.5
            kk[:, :, 0] = (120.0 * (torch.arange(cap) + 1) / cap)[:, None]
            k[s * cap:(s + 1) * cap] = kk.reshape(cap, -1)
    seqs, targets, k0s, qs = [], [], [], 0
    for b, (sq, sk) in enumerate(pairs):
        k0 = (nkv - b // share) * cap
        if mode == "decoy":
            qc, t = H.decoy_query_code(sq, sk, causal, 1, hq, hd)
            q[qs:qs + sq] = qc.reshape(sq, -1)
            targets.append(k0 + t)
        else:
            qq = torch.randn(sq, hq, hd, generator=gen)
            qq[:, :, 0] = 8.0
            q[qs:qs + sq] = qq.reshape(sq, -1)
        i = torch.arange(sq)
        seqs.append((qs + i, k0 + torch.arange(sk), i + sk - sq + 1 if causal else torch.full((sq,), sk)))
        k0s.append(k0)
        qs += sq
    if nan_rest:
        keep = torch.zeros(slots * cap, dtype=torch.bool)
        for (_, sk), k0 in zip(pairs, k0s):
            keep[k0:k0 + sk] = True
        k[~keep], v[~keep] = float("nan"), float("nan")
    q, k, v = (x.to(torch.bfloat16) for x in (q, k, v))
    expect = H.decoy_expect(v, torch.cat(targets), hq // hkv, hd) if mode == "decoy" else None
    return q, k, v, seqs, expect, k0s, cap


FORMS = {   # name -> (query / key lengths per sequence, causal)
    "self": ([(1, 1), (63, 63), (64, 64), (65, 65), (130, 130)], True),
    "self_noncausal": ([(33, 33), (65, 65), (130, 130)], False),
    "decode": ([(1, 1), (1, 64), (5, 65), (5, 129), (1, 300)], True),
    "chunk": ([(17, 17 + 63), (18, 18 + 64), (65, 65 + 321), (1, 1 + 320)], True),
    "cross": ([(32, 4), (8, 49), (1, 64), (17, 200)], False),
}


@pytest.mark.parametrize("form", sorted(FORMS))
@pytest.mark.parametrize("hd", [48, 64, 80, 128])
def test_decoys_separate_the_target_by_20_nats_and_the_reference_is_exact(hd, form):
    """For every (row, head): the target beats every other visible key by more than 20 nats, keys of the opposite
    parity (a neighbouring packed sequence) beat it by more than 20 nats, and so do zero rows; causal rows that have a
    key i + 1 see it beat the target by more than 20 nats in most cases.  The float64 softmax rounds to exactly the
    expected V rows."""
    pairs, causal = FORMS[form]
    hkv, group = 2, 2
    hq = hkv * group
    q, k, v, seqs, expect, _, cap = _pool(pairs, hd, hq, hkv, causal, "decoy")
    scale = H.decoy_scale(hd)
    decoys = rows_with_next = 0
    for (q_rows, k_rows, vis), (sq, sk) in zip(seqs, pairs):
        qc, t = H.decoy_query_code(sq, sk, causal, 1, hq, hd)
        kc = H.decoy_key_code(sk + 1, 1, hd)                       # the sequence's keys and the one after them
        s = torch.einsum("ihd,jd->ihj", qc.double(), kc.double()) * scale
        j = torch.arange(sk + 1)[None, None, :]
        visible = j < vis[:, None, None]
        st = s.gather(2, t[:, :, None])
        others = s.masked_fill(~visible | (j == t[:, :, None]), -float("inf")).amax(2)
        assert bool((st[:, :, 0] - others > 20).all()), (hd, form, float((st[:, :, 0] - others).min()))
        opposite = torch.einsum("ihd,jd->ihj", qc.double(), H.decoy_key_code(sk, -1, hd).double()) * scale
        assert bool((opposite.amin(2) - st[:, :, 0] > 20).all())
        assert bool((-st > 20).all())                              # a zero row scores 0
        if causal:
            nxt = vis < sk + 1                                     # rows with a hidden key right after their diagonal
            s_next = s[torch.arange(sq), :, vis.clamp(max=sk)]
            decoys += int(((s_next - st[:, :, 0] > 20) & nxt[:, None]).sum())
            rows_with_next += int(nxt.sum()) * hq
    if causal and rows_with_next:
        assert decoys >= 0.4 * rows_with_next, (decoys, rows_with_next)
    out, _, _ = H.attention_ref_rows(q, k, v, seqs, hkv, group, scale, hd)
    assert torch.equal(out.to(torch.bfloat16).view(torch.int16), expect.view(torch.int16))


# ------------------------------------------------------------------------------------------ mutations
def _shift_vis(d):
    return lambda seqs, ctx: [(qr, kr, (vis + d).clamp(0, kr.numel())) for qr, kr, vis in seqs]


def _k_len(d):
    def f(seqs, ctx):
        out = []
        for qr, kr, vis in seqs:
            sk, sq = kr.numel() + d, qr.numel()
            out.append((qr, kr[0] + torch.arange(sk), (torch.arange(sq) + sk - sq + 1).clamp(0, sk)))
        return out
    return f


def _row0(d):
    return lambda seqs, ctx: [(qr, kr + d, vis) for qr, kr, vis in seqs]


def _next_env(seqs, ctx):
    k0s = sorted({int(kr[0]) for _, kr, _ in seqs})
    nxt = {a: b for a, b in zip(k0s, k0s[1:] + k0s[:1])}
    return [(qr, kr - kr[0] + nxt[int(kr[0])], vis) for qr, kr, vis in seqs]


def _drop_last_block(seqs, ctx):
    return [(qr, kr, vis.clamp(max=64 * (kr.numel() // 64))) for qr, kr, vis in seqs]


def _ctx_zero(seqs, ctx):
    return [(qr, kr[:qr.numel()], torch.arange(qr.numel()) + 1) for qr, kr, vis in seqs]


# name -> (layout: pairs, causal, kv_div[, NaN past the keys]; wrong reference).  A non-causal row past k_len scores
# no higher than the other hidden keys, so k_len + 1 is caught there by the NaN the pools hold past k_len.
MUTATIONS = {
    "causal_offset_plus_1": (([(5, 70), (65, 130)], True, 1), _shift_vis(1)),
    "causal_offset_minus_1": (([(5, 70), (65, 130)], True, 1), _shift_vis(-1)),
    "k_len_plus_1": (([(1, 64), (5, 129), (1, 200)], True, 1), _k_len(1)),
    "k_len_minus_1": (([(1, 64), (5, 129), (1, 200)], True, 1), _k_len(-1)),
    "k_len_plus_1_noncausal": (([(8, 33), (8, 33)], False, 2, True), _k_len(1)),
    "row0_plus_1": (([(5, 65), (1, 130)], True, 1), _row0(1)),
    "row0_minus_1": (([(5, 65), (1, 130)], True, 1), _row0(-1)),
    "kv_div_next_env": (([(8, 34)] * 6, False, 3), _next_env),
    "last_partial_block_dropped": (([(1, 65), (17, 150), (5, 200)], True, 1), _drop_last_block),
    "last_partial_block_dropped_noncausal": (([(32, 100), (8, 49)], False, 1), _drop_last_block),
    "ctx_zero": (([(17, 17 + 64), (18, 18 + 321)], True, 1), _ctx_zero),
}


@pytest.mark.parametrize("name", sorted(MUTATIONS) + ["gqa_head_map_mod"])
@pytest.mark.parametrize("hd", [48, 128])
def test_exact_check_and_bound_reject_a_wrong_reference(hd, name):
    """The correct reference passes both checks; the wrong one fails the exact decoy check and the float64 bound."""
    hkv, group = 2, 2
    if name == "gqa_head_map_mod":
        layout, wrong = ([(5, 70), (64, 64)], True, 1), (lambda seqs, ctx: seqs)
        head_map = lambda h: h % hkv
    else:
        layout, wrong = MUTATIONS[name]
        head_map = None
    pairs, causal, share = layout[:3]
    nan_rest = len(layout) > 3 and layout[3]
    hq = hkv * group
    # decoys: the wrong reference misses the expected V somewhere
    q, k, v, seqs, expect, _, _ = _pool(pairs, hd, hq, hkv, causal, "decoy", share, nan_rest=nan_rest)
    scale = H.decoy_scale(hd)
    good, _, _ = H.attention_ref_rows(q, k, v, seqs, hkv, group, scale, hd)
    assert not bool((good.to(torch.bfloat16).view(torch.int16) != expect.view(torch.int16)).any())
    bad, _, _ = H.attention_ref_rows(q, k, v, wrong(seqs, None), hkv, group, scale, hd, head_map=head_map)
    assert bool((bad.to(torch.bfloat16).view(torch.int16) != expect.view(torch.int16)).any()), name + ": exact check"
    # random rising-maximum data: the wrong reference leaves attention_bound of the right one
    q, k, v, seqs, _, _, _ = _pool(pairs, hd, hq, hkv, causal, "random", share, seed=1, nan_rest=nan_rest)
    ref, mag, dl = H.attention_ref_rows(q, k, v, seqs, hkv, group, SCALE, hd)
    keys = max(sk for _, sk in pairs)
    bound = H.attention_bound(ref, mag, dl, group, hd, keys)
    assert not bool(H.bound_violations(ref.to(torch.bfloat16), ref, bound)[0].any())
    wr, _, _ = H.attention_ref_rows(q, k, v, wrong(seqs, None), hkv, group, SCALE, hd, head_map=head_map)
    assert bool(H.bound_violations(wr.to(torch.bfloat16), ref, bound)[0].any()), name + ": bound"
