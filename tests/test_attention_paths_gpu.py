"""Every forward attention path besides the head-dim-128 var-len wgmma prefill, held to the standard of
tests/test_hopper_kernels_gpu.py:

  * slotted K/V cache decode (hd 128, GQA, q a column slice of the packed q|k|v rows, permuted pool slots, k_len at
    every 64-key edge up to 2048) and the NavDP critic's slotted cross-attention (hd 48, kv_div, K/V base past the
    masked rows);
  * the chunk continuation over a K/V pool (attention_cache_wgmma.cu) at every GQA group size;
  * the generic mma.sync kernel at hd 48 / 64 / 80 / 128 (fixed, var-len, kv_div cross-attention);
  * the short-sequence kernel at every key-tile count and query-sequence grouping.

Each path is checked twice: exact decoys (every (row, head) output must be exactly its target key's V) and random data
whose softmax maximum rises from key block to key block, against the float64 softmax with attention_bound.  Every call
runs twice and must reproduce itself bit for bit; every output is a view in a sentinel-filled buffer with a wider row
stride, and the sentinels must survive; the kernel the library reports having routed the call to must be the one the
case is for.  Pool and slot rows a kernel must never read hold NaN, so any read of one shows in the output (0 * NaN is
NaN); neighbouring sequences of packed buffers are real data of the opposite decoy parity.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_hopper_kernels_gpu as H  # noqa: E402

pytestmark = pytest.mark.gpu
NAN = float("nan")
RAND_SCALE = 0.0625


@pytest.fixture(scope="module")
def L():
    from internnav_b200 import _lib
    _lib.lib()
    return _lib


# ------------------------------------------------------------------------------------------ case construction
class Case:
    """Buffers and sequences of one attention call.

    q / k / v are column slices (q_cols, k_cols, v_cols) of float32 staging buffers, NaN wherever no sequence puts data.
    seqs: one (q_rows, k_start, sk, sigma) per query sequence: its query rows, the first of its sk key rows (K/V shared
    by several query sequences are listed by each) and its decoy parity.  launch(L, q, k, v, o) runs the call on the
    bf16 CUDA views and returns the reported route (None for attention_cache, which has one kernel)."""

    def __init__(self, hd, hq, hkv, causal, q_shape, q_cols, kv_shape, k_cols, v_cols, seqs, launch, kv_same=False,
                 v_shape=None):
        self.hd, self.hq, self.hkv, self.causal = hd, hq, hkv, causal
        self.qbuf = torch.full(q_shape, NAN)
        self.kbuf = self.qbuf if kv_same else torch.full(kv_shape, NAN)
        self.vbuf = torch.full(v_shape, NAN) if v_shape else self.kbuf   # V in a buffer of its own (a third stride)
        self.q_cols, self.k_cols, self.v_cols = q_cols, k_cols, v_cols
        self.seqs, self.launch = seqs, launch
        self.scale = None   # set while the random data runs; launches use _scale(case)

    def _views(self, qb, kb, vb):
        c = lambda b, c0, n: b[:, c0:c0 + n]
        return (c(qb, self.q_cols, self.hq * self.hd), c(kb, self.k_cols, self.hkv * self.hd),
                c(vb, self.v_cols, self.hkv * self.hd))

    def _device(self):
        done = {}
        dev = lambda b: done.setdefault(id(b), b.to(torch.bfloat16).cuda())
        return self._views(dev(self.qbuf), dev(self.kbuf), dev(self.vbuf))

    def fill(self, mode, seed):
        """Writes decoys or random data; -> (q, k, v) bf16 CUDA views and, for decoys, (expect, key_rows, kstart, klen)
        per query row in the order of the concatenated q_rows."""
        gen = torch.Generator().manual_seed(seed)
        q, k, v = self._views(self.qbuf, self.kbuf, self.vbuf)
        hd, hq, hkv = self.hd, self.hq, self.hkv
        done = set()
        key_rows, kstart, klen = [], [], []
        for q_rows, k0, sk, sigma in self.seqs:
            sq = len(q_rows)
            if k0 not in done:
                done.add(k0)
                if mode == "decoy":
                    k[k0:k0 + sk] = H.decoy_key_code(sk, sigma, hd).repeat(1, hkv)
                    v[k0:k0 + sk] = H.decoy_values(sk, hkv * hd, gen)
                else:   # dim 0 of each head: a ramp to 60 nats (8 * 120 * 0.0625) at the sequence's last key
                    kk = torch.randn(sk, hkv, hd, generator=gen) * 1.5
                    kk[:, :, 0] = (120.0 * (torch.arange(sk) + 1) / sk)[:, None]
                    k[k0:k0 + sk] = kk.reshape(sk, -1)
                    v[k0:k0 + sk] = torch.randn(sk, hkv * hd, generator=gen)
            if mode == "decoy":
                qc, t = H.decoy_query_code(sq, sk, self.causal, sigma, hq, hd)
                q[q_rows] = qc.reshape(sq, -1)
                key_rows.append(k0 + t)
                kstart.append(torch.full((sq,), k0))
                klen.append(torch.full((sq,), sk))
            else:
                qq = torch.randn(sq, hq, hd, generator=gen)
                qq[:, :, 0] = 8.0
                q[q_rows] = qq.reshape(sq, -1)
        views = self._device()
        if mode != "decoy":
            return views, None
        key_rows = torch.cat(key_rows)
        return views, (H.decoy_expect(views[2], key_rows, hq // hkv, hd).cuda(), key_rows, torch.cat(kstart),
                       torch.cat(klen))

    def q_rows(self):
        return torch.cat([torch.as_tensor(r) for r, _, _, _ in self.seqs])

    def ref_seqs(self):
        out = []
        for q_rows, k0, sk, _ in self.seqs:
            sq = len(q_rows)
            i = torch.arange(sq)
            vis = i + sk - sq + 1 if self.causal else torch.full((sq,), sk)
            out.append((torch.as_tensor(q_rows).cuda(), (k0 + torch.arange(sk)).cuda(), vis.cuda()))
        return out


def _run_twice(L, case, views, what):
    q, k, v = views
    outs, routes = [], []
    for _ in range(2):
        buf, o = H.guarded(case.qbuf.shape[0], case.hq * case.hd, torch.bfloat16, "cuda", top=1, bottom=4, left=64,
                           right=72)
        routes.append(case.launch(L, q, k, v, o))
        torch.cuda.synchronize()
        H.assert_guard(buf, o, what)
        outs.append(o.clone())
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), what + ": second call differs"
    assert routes[0] == routes[1]
    return outs[0], routes[0]


def check_case(L, case, route, what, seed=0):
    """Exact decoys, then bounded random data, on the same layout; `route` is the kernel the call must report."""
    views, (expect, key_rows, kstart, klen) = case.fill("decoy", seed)
    o, got = _run_twice(L, case, views, what + " decoys")
    assert got == route, "%s: routed to %s, expected %s" % (what, got, route)
    rows = case.q_rows().cuda()
    o = o[rows]
    hq, hd, group = case.hq, case.hd, case.hq // case.hkv
    bad = (o.view(torch.int16) != expect.view(torch.int16)).view(-1, hq, hd).any(-1)
    if bool(bad.any()):
        r, h = (int(x) for x in bad.nonzero()[0])
        saw = H.identify_key(o[r, h * hd:(h + 1) * hd], views[2], 0, h // group, hd=hd,
                             rows=torch.arange(int(kstart[r]), int(kstart[r] + klen[r])))
        raise AssertionError("%s: %d of %d (row, head) outputs wrong; first: query row %d (buffer row %d) head %d should "
                             "see key %d only, saw %s" % (what, int(bad.sum()), bad.numel(), r, int(rows[r]), h,
                                                          int(key_rows[r, h] - kstart[r]), saw))
    views, _ = case.fill("random", seed + 1)
    q, k, v = views
    case.scale = RAND_SCALE
    try:
        o, got = _run_twice(L, case, views, what + " random")
    finally:
        case.scale = None
    ref, mag, dl = H.attention_ref_rows(q, k, v, case.ref_seqs(), case.hkv, group, RAND_SCALE, hd)
    assert float(dl.max()) < 1e-3
    keys = max(sk for _, _, sk, _ in case.seqs)
    H.assert_within(o[rows], ref, H.attention_bound(ref, mag, dl, group, hd, keys), what + " random")


def _scale(case):
    """The call's softmax scale: the decoys' one score unit = 8 nats, or the random data's 0.0625."""
    return case.scale or H.decoy_scale(case.hd)


def _i32(x):
    return torch.tensor(x, dtype=torch.int32, device="cuda")


# ------------------------------------------------------------------------------------------ slotted decode, hd 128
DECODE_KLEN = [1, 63, 64, 65, 127, 128, 129, 2047, 2048]


@pytest.mark.parametrize("addressing", ["row0", "slot"])
@pytest.mark.parametrize("hq,hkv", [(28, 4), (2, 1)])
@pytest.mark.parametrize("per_seq", [1, 5])
def test_slotted_decode(L, per_seq, hq, hkv, addressing):
    """System 2's decode step / latent pass (s2_model.cu chunk_pass): per_seq new rows per sequence, q the query columns
    of the packed q|k|v rows, K/V in pool slots (permuted through k_row0, or sequence b at slot b * k_slot), the cache
    lengths at every 64-key edge up to 2048 in one launch, bottom-right causal."""
    hd, cap = 128, 2048 + 64
    klen = [max(n, per_seq) for n in DECODE_KLEN]
    B = len(klen)
    slots = [(3 * b + 2) % (B + 1) for b in range(B)] if addressing == "row0" else list(range(B))
    qkv_n = (hq + 2 * hkv) * hd
    seqs = [(torch.arange(b * per_seq, (b + 1) * per_seq), slots[b] * cap, klen[b], 1) for b in range(B)]
    kl, r0 = _i32(klen), _i32([s * cap for s in slots])

    def launch(L, q, k, v, o):
        return L.attention_test(q, k, v, o, hq, hkv, hd, B, seq_q=per_seq, causal=True, scale=_scale(c), k_len=kl,
                                k_slot=cap, k_row0=r0 if addressing == "row0" else None)
    c = Case(hd, hq, hkv, True, (B * per_seq, qkv_n), 0, ((B + 1) * cap, 2 * hkv * hd), 0, hkv * hd, seqs, launch)
    check_case(L, c, ("generic", 128, 0, 1), "decode per_seq=%d %d/%d %s" % (per_seq, hq, hkv, addressing))


# ------------------------------------------------------------------------------------------ slotted critic, hd 48
@pytest.mark.parametrize("T", [8, 32])
def test_slotted_critic_cross_attention(L, T):
    """The NavDP critic's cross-attention (s1_model.cu): the K/V base advanced by kv_first rows past the masked time /
    goal slots, environment e's keys at e * Mtok (k_slot = Mtok) with k_len < Mtok of them, kv_div = Ns trajectories per
    environment, K and V interleaved in the per-layer condition buffer, non-causal."""
    hd, heads, D = 48, 8, 384
    Benv, Ns, Mtok, kv_first = 3, 4, 40, 2
    klen = [38, 17, 1]
    ldkv = 4 * D                                   # two layers of K | V; layer 1 is used
    seqs = [(torch.arange(b * T, (b + 1) * T), (b // Ns) * Mtok + kv_first, klen[b // Ns], 1) for b in range(Benv * Ns)]
    kl = _i32(klen)

    def launch(L, q, k, v, o):
        return L.attention_test(q, k[kv_first:], v[kv_first:], o, heads, heads, hd, Benv * Ns, seq_q=T, seq_k=max(klen),
                                kv_div=Ns, causal=False, scale=_scale(c), k_len=kl, k_slot=Mtok)
    c = Case(hd, heads, heads, False, (Benv * Ns * T, D), 0, (Benv * Mtok, ldkv), 2 * D, 3 * D, seqs, launch)
    check_case(L, c, ("generic", 48, 0, 1), "critic T=%d" % T)


# ------------------------------------------------------------------------------------------ chunk continuation
CONT_CTX = [0, 1, 63, 64, 319, 320, 321, 2047]
CONT_N = [1, 17, 18, 63, 64, 65, 400]      # 18 = 2 R at G = 7: one whole query tile


@pytest.mark.parametrize("group", [1, 2, 3, 4, 7, 8, 64])
@pytest.mark.parametrize("ctx", CONT_CTX)
def test_chunk_continuation(L, ctx, group):
    """The look-down turn's prefill over a K/V pool (attention_cache_wgmma.cu): chunks of every length of CONT_N after
    ctx cached rows, plus a shorter neighbour at ctx // 3, in one launch (slots permuted, rows past ctx + n of a slot
    NaN); one sequence with no new rows between two others; q the query columns of the packed q|k|v rows with the last
    sequence's query tile running past the buffer's end; the output a guarded view.  G = heads_q / heads_kv query heads
    share a K / V head (64 % G != 0 for 3 and 7)."""
    hd = 128
    hkv = {7: 4, 64: 1}.get(group, 2)
    hq = hkv * group
    shapes = [(ctx, n) for n in CONT_N if n != 65]
    shapes.insert(len(shapes) // 2, (100, 0))       # no new rows
    shapes += [(ctx // 3, 5), (ctx, 65)]            # 65 rows last: its query tile is partial at every G
    assert shapes[-1][1] % (2 * (64 // group)) != 0
    B = len(shapes)
    # slots of ctx + n + 64 rows in a permuted order; the 64 rows past each sequence's keys stay NaN
    order = sorted(range(B), key=lambda b: (5 * b + 3) % B)
    row0, r = [0] * B, 0
    for b in order:
        row0[b], r = r, r + sum(shapes[b]) + 64
    cu = [0]
    for _, n in shapes:
        cu.append(cu[-1] + n)
    seqs = [(torch.arange(cu[b], cu[b + 1]), row0[b], c + n, 1) for b, (c, n) in enumerate(shapes) if n > 0]
    cu_t, ctx_t, row0_t = _i32(cu), _i32([c for c, _ in shapes]), _i32(row0)
    qkv_n = (hq + 2 * hkv) * hd

    def launch(L, q, k, v, o):
        L.attention_cache(q, k, v, hq, hkv, cu_t, ctx_t, row0_t, max(n for _, n in shapes), scale=_scale(c), out=o)
        return None
    c = Case(hd, hq, hkv, True, (cu[-1], qkv_n), 0, (r, 2 * hkv * hd), 0, hkv * hd, seqs, launch)
    check_case(L, c, None, "continuation ctx=%d G=%d" % (ctx, group), seed=ctx + group)


# ------------------------------------------------------------------------------------------ generic kernel
def _packed(pairs, gap=0):
    """Query / key row starts of sequences (sq, sk) packed back to back -> (q starts, k starts, q rows, k rows)."""
    qs, ks = [0], [0]
    for sq, sk in pairs:
        qs.append(qs[-1] + sq)
        ks.append(ks[-1] + sk)
    return qs, ks, qs[-1] + gap, ks[-1] + gap


def _varlen_case(hd, hq, hkv, causal, lens, total_rows=0, tail=7):
    """Var-len self-attention over packed rows (cu_q = cu_k), consecutive sequences of opposite parity, NaN rows past the
    last sequence."""
    qs, _, rows, _ = _packed([(n, n) for n in lens], tail)
    seqs = [(torch.arange(qs[b], qs[b + 1]), qs[b], n, 1 if b % 2 == 0 else -1) for b, n in enumerate(lens)]
    cu = _i32(qs)

    def launch(L, q, k, v, o):
        return L.attention_test(q, k, v, o, hq, hkv, hd, len(lens), cu_q=cu, cu_k=cu, max_seq_q=max(lens),
                                causal=causal, scale=_scale(c), total_rows=total_rows)
    c = Case(hd, hq, hkv, causal, (rows, hq * hd), 0, (rows, 2 * hkv * hd), 0, hkv * hd, seqs, launch)
    return c


def _boundary_lengths(hd):
    lim = H.decoy_max_keys(hd)
    lens = {1, lim - 1, lim}
    for m in range(1, lim // 64 + 1):
        lens |= {64 * m - 1, 64 * m, 64 * m + 1}
    return sorted(x for x in lens if x <= lim)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("hd", [48, 64, 80, 128])
def test_generic_fixed_length(L, hd, causal):
    """Fixed-length batches (no cu_seqlens): three packed sequences of 130 rows, two query heads per K/V head."""
    n, B, hkv, hq = 130, 3, 2, 4
    seqs = [(torch.arange(b * n, (b + 1) * n), b * n, n, 1 if b % 2 == 0 else -1) for b in range(B)]

    def launch(L, q, k, v, o):
        return L.attention_test(q, k, v, o, hq, hkv, hd, B, seq_q=n, seq_k=n, causal=causal, scale=_scale(c))
    c = Case(hd, hq, hkv, causal, (B * n, hq * hd), 0, (B * n, 2 * hkv * hd), 0, hkv * hd, seqs, launch)
    check_case(L, c, ("generic", hd, 0, 1), "fixed hd=%d causal=%s" % (hd, causal))


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("hd", [48, 64, 80, 128])
def test_generic_varlen_every_boundary(L, hd, causal):
    """Var-len, the sequence lengths at every 64-key edge up to the longest exact decoy sequence of the head dim (480 /
    992 / 960 / 4032).  At hd 128 the call carries total_rows like the System-2 prefill, and its sequences past 320
    keys keep it on the generic kernel."""
    lens = _boundary_lengths(hd)
    hq, hkv = (2, 1) if hd == 128 else (4, 2)
    c = _varlen_case(hd, hq, hkv, causal, lens, total_rows=sum(lens) + 7 if hd == 128 else 0)
    check_case(L, c, ("generic", hd, 0, 1), "varlen hd=%d causal=%s" % (hd, causal))


def test_generic_hd128_prefill_past_320(L):
    """The System-2 prefill of a batch with one prompt longer than 320 tokens (28 / 4 heads, total_rows given)."""
    lens = [200, 321, 64, 777]
    c = _varlen_case(128, 28, 4, True, lens, total_rows=sum(lens) + 7)
    check_case(L, c, ("generic", 128, 0, 1), "hd128 prefill past 320")


def test_generic_hd64_kv_div_three_strides(L):
    """The NextDiT cross-attention (hd 64): each K/V sequence shared by kv_div = 3 query sequences, q, k and v at three
    different row strides."""
    hd, heads, B, kv_div, sq, sk = 64, 4, 6, 3, 33, 77
    nkv = B // kv_div
    seqs = [(torch.arange(b * sq, (b + 1) * sq), (b // kv_div) * sk, sk, 1 if (b // kv_div) % 2 == 0 else -1)
            for b in range(B)]

    def launch(L, q, k, v, o):
        assert len({q.stride(0), k.stride(0), v.stride(0)}) == 3
        return L.attention_test(q, k, v, o, heads, heads, hd, B, seq_q=sq, seq_k=sk, kv_div=kv_div, scale=_scale(c))
    c = Case(hd, heads, heads, False, (B * sq, heads * hd + 64), 64, (nkv * sk, 2 * heads * hd), 0, 0, seqs, launch,
             v_shape=(nkv * sk, heads * hd + 128))
    check_case(L, c, ("generic", 64, 0, 1), "hd64 kv_div")


def test_generic_hd48_qformer_cross_1024(L):
    """The Q-former cross-attention: 32 queries over 1024 keys, 8 heads of 48 (past the exact decoy limit: bounded
    random data only)."""
    hd, heads, B, sq, sk = 48, 8, 3, 32, 1024
    _bounded_only(L, hd, heads, heads, False, [(b * sq, sq, b * sk, sk) for b in range(B)], B * sq, B * sk,
                  lambda L, q, k, v, o, s: L.attention_test(q, k, v, o, heads, heads, hd, B, seq_q=sq, seq_k=sk,
                                                            scale=s),
                  ("generic", 48, 0, 1), "qformer cross")


def test_generic_hd80_vit_windows_and_full(L):
    """Qwen ViT attention (hd 80, 16 heads, var-len): windows of 64 and 41 tokens plus one full-attention sequence of
    1200 (past the exact decoy limit: bounded random data only)."""
    lens = [64, 64, 41, 64, 1200, 64]
    hd, heads = 80, 16
    qs, _, rows, _ = _packed([(n, n) for n in lens])
    cu = _i32(qs)
    _bounded_only(L, hd, heads, heads, False, [(qs[b], n, qs[b], n) for b, n in enumerate(lens)], rows, rows,
                  lambda L, q, k, v, o, s: L.attention_test(q, k, v, o, heads, heads, hd, len(lens), cu_q=cu, cu_k=cu,
                                                            max_seq_q=max(lens), scale=s),
                  ("generic", 80, 0, 1), "vit windows + full")


def _bounded_only(L, hd, hq, hkv, causal, spans, q_rows, k_rows, call, route, what):
    """Random rising-maximum data only, for shapes past the exact decoy limit: spans = [(q0, sq, k0, sk)]."""
    seqs = [(torch.arange(q0, q0 + sq), k0, sk, 1) for q0, sq, k0, sk in spans]
    c = Case(hd, hq, hkv, causal, (q_rows, hq * hd), 0, (k_rows, 2 * hkv * hd), 0, hkv * hd, seqs,
             lambda L, q, k, v, o: call(L, q, k, v, o, RAND_SCALE))
    views, _ = c.fill("random", 3)
    o, got = _run_twice(L, c, views, what)
    assert got == route, "%s: routed to %s, expected %s" % (what, got, route)
    ref, mag, dl = H.attention_ref_rows(*views, c.ref_seqs(), hkv, hq // hkv, RAND_SCALE, hd)
    assert float(dl.max()) < 1e-3
    keys = max(s[3] for s in spans)
    H.assert_within(o[c.q_rows().cuda()], ref, H.attention_bound(ref, mag, dl, hq // hkv, hd, keys), what)


def test_hd48_odd_output_stride_leaves_the_short_kernel(L):
    """A call the short-sequence kernel would take, but into an output whose row stride is 2 (mod 8): its 16-byte
    stores cannot serve it, so it must run on the generic kernel, exactly, with the guard band intact."""
    hd, heads, B, n = 48, 8, 4, 8
    seqs = [(torch.arange(b * n, (b + 1) * n), b * n, n, 1 if b % 2 == 0 else -1) for b in range(B)]
    c = Case(hd, heads, heads, True, (B * n, heads * hd), 0, (B * n, 2 * heads * hd), 0, heads * hd, seqs, None)
    views, (expect, _, _, _) = c.fill("decoy", 0)
    outs = []
    for _ in range(2):
        buf, o = H.guarded(B * n, heads * hd, torch.bfloat16, "cuda", left=8, right=10)
        assert o.stride(0) % 8 == 2
        got = L.attention_test(*views, o, heads, heads, hd, B, seq_q=n, seq_k=n, causal=True, scale=H.decoy_scale(hd))
        torch.cuda.synchronize()
        assert got == ("generic", 48, 0, 1), got
        H.assert_guard(buf, o, "ldo % 8 = 2")
        outs.append(o.clone())
    assert torch.equal(outs[0].view(torch.int16), expect.view(torch.int16)), "ldo % 8 = 2: decoys not exact"
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), "ldo % 8 = 2: second call differs"


# ------------------------------------------------------------------------------------------ short-sequence kernel
SHORT_SK = [4, 16, 17, 33, 34, 49, 64]        # 16-key tiles 1, 1, 2, 3, 3, 4, 4
SHORT_SQ = [1, 8, 17, 32]
SHORT_KV_DIV = [(1, 5), (3, 6), (2, 6), (4, 8)]   # (kv_div, batch): G = 1, 1, 2, 4


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("sk", SHORT_SK)
def test_short_kernel(L, sk, causal):
    """The short-sequence kernel (hd 48, 8 heads): every query length of SHORT_SQ against sk keys, with kv_div such that
    1, 2 and 4 query sequences share a CTA.  Non-causal: the cross layout (K and V interleaved in one condition buffer,
    each K/V sequence shared by kv_div query sequences).  Causal: the self-attention layout (q, k, v column slices of
    packed q|k|v rows) where sq = sk, else bottom-right causal over the cross layout."""
    hd, heads, D = 48, 8, 384
    nkp = (sk + 15) // 16
    for sq in SHORT_SQ:
        if causal and sq > sk:
            continue
        for kv_div, B in SHORT_KV_DIV:
            G = 4 if kv_div % 4 == 0 and B % 4 == 0 else 2 if kv_div % 2 == 0 and B % 2 == 0 else 1
            what = "short sq=%d sk=%d kv_div=%d B=%d causal=%s" % (sq, sk, kv_div, B, causal)
            if causal and sq == sk and kv_div == 1:
                seqs = [(torch.arange(b * sq, (b + 1) * sq), b * sk, sk, 1 if b % 2 == 0 else -1) for b in range(B)]

                def launch(L, q, k, v, o, B=B, sq=sq, kv_div=kv_div):
                    return L.attention_test(q, k, v, o, heads, heads, hd, B, seq_q=sq, seq_k=sq, kv_div=kv_div,
                                            causal=True, scale=_scale(c))
                c = Case(hd, heads, heads, True, (B * sq, 3 * D), 0, None, D, 2 * D, seqs, launch, kv_same=True)
            else:
                nkv = B // kv_div
                seqs = [(torch.arange(b * sq, (b + 1) * sq), (b // kv_div) * sk, sk, 1 if (b // kv_div) % 2 == 0 else -1)
                        for b in range(B)]

                def launch(L, q, k, v, o, B=B, sq=sq, kv_div=kv_div):
                    return L.attention_test(q, k, v, o, heads, heads, hd, B, seq_q=sq, seq_k=sk, kv_div=kv_div,
                                            causal=causal, scale=_scale(c))
                c = Case(hd, heads, heads, causal, (B * sq, D), 0, (nkv * sk, 2 * D), 0, D, seqs, launch)
            check_case(L, c, ("short", 48, nkp, G), what, seed=sq + sk)
