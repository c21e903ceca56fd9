"""Tile-edge tests of the four Hopper tensor-core kernels (gemm_wgmma.cu, wgrad_tn.cu, attention_wgmma.cu, ff_block.cu).

Each case compares the kernel with a float64 reference of the same operation, element by element:
  * exact cases draw every operand from small integers, so the fp32 accumulation is exact in any order and the kernel
    must equal the float64 result rounded once to the output type, bit for bit;
  * the rest (GELU / tanh-GELU / SiLU / SwiGLU epilogues, softmax, LayerNorm) are held to `elementwise_bound`;
  * every output is a view inside a larger buffer filled with a sentinel bit pattern (rows below and above, columns on
    both sides, a row stride wider than the row), and the sentinels must survive the call;
  * a second identical call must reproduce the first bit for bit (all four kernels reduce in a fixed order).

The helpers above the tests take CPU or CUDA tensors; tests/test_kernel_checks_host.py feeds them deliberately wrong
references on the CPU to show that they reject the errors these tests exist for.
"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32 = 2.0 ** -24        # unit roundoff of fp32
BF16_U = 2.0 ** -8      # unit roundoff of bf16 (8-bit significand): half an ulp is at most 2^-8 of the value
ACT_NONE, ACT_GELU, ACT_RELU, ACT_SWIGLU, ACT_GELU_TANH, ACT_SILU = 0, 1, 2, 3, 4, 5


# ------------------------------------------------------------------------------------------ shared checks
def small_ints(shape, lo, hi, gen, dtype=torch.bfloat16, device="cpu"):
    """Integers drawn uniformly from [lo, hi], exactly representable in `dtype`."""
    return torch.randint(lo, hi + 1, tuple(shape), generator=gen).to(dtype).to(device)


def exact_mismatches(out, ref64):
    """Elements where `out` differs from the float64 result rounded once to out's dtype -> (bool mask, expected).

    The premise of the exact cases is checked here too: every reference value must be an fp32 value, so that the
    float64 -> bf16 conversion is a single rounding and any fp32 accumulation order gives the same number."""
    ref64 = ref64.to(torch.float64)
    assert torch.equal(ref64.float().double(), ref64), "exact reference leaves fp32: operands too large"
    want = ref64.to(out.dtype)
    if out.dtype == torch.bfloat16:   # compare bit patterns, so -0 / +0 and NaNs are told apart
        bad = out.view(torch.int16) != want.view(torch.int16)
    else:
        bad = out.view(torch.int32) != want.view(torch.int32)
    return bad, want


def assert_exact(out, ref64, what):
    bad, want = exact_mismatches(out, ref64)
    if bool(bad.any()):
        idx = bad.nonzero()[:5].tolist()
        shown = ", ".join("%s got %r want %r" % (tuple(i), out[tuple(i)].item(), want[tuple(i)].item()) for i in idx)
        raise AssertionError("%s: %d of %d elements differ from the exact result; first: %s"
                             % (what, int(bad.sum()), bad.numel(), shown))


def elementwise_bound(ref, mag, k, extra=0.0, bf16_out=True):
    """Largest |kernel - ref| allowed per element, ref the float64 value of the same operation on the same inputs.

      2^-8 (|ref| + e)     the output's single rounding to bf16 (half an ulp never exceeds 2^-8 of the value), applied to
                           the value the kernel holds in fp32, which may differ from ref by e, the rest of this bound;
      (k + 64) 2^-24 mag   fp32 arithmetic.  `mag` is the same computation on absolute values (for a dot product
                           sum |a||w|, then through bias, activation, scale and residual); a k-term fp32 sum in any order
                           is within (k - 1) 2^-24 sum |terms| of the exact sum (Higham, Accuracy and Stability of
                           Numerical Algorithms, eq. 3.5).  The 64 units cover the epilogue: a handful of roundings of
                           the bias / scale / residual, and the activations -- the GELU's erf polynomial is within 3e-7
                           (5 units) and its reciprocal's ~2-unit error is raised to the 16th power (<= 40 units of |v|
                           after the 0.5 v factor); tanhf, __expf and __fdividef stay within a few units;
      extra                known, separately bounded errors that are not fp32 rounding: bf16 roundings of intermediate
                           operands (P in the attention, the LayerNorm output and hidden activations of the FF block).
    """
    e = (k + 64) * U32 * mag + extra
    return BF16_U * (ref.abs() + e) + e if bf16_out else e


def bound_violations(out, ref, bound):
    """(bool mask of elements outside the bound, |out - ref|)."""
    err = (out.to(torch.float64) - ref).abs()
    return ~(err <= bound), err


def assert_within(out, ref, bound, what):
    bad, err = bound_violations(out, ref, bound)
    if bool(bad.any()):
        idx = bad.nonzero()[:5].tolist()
        shown = ", ".join("%s got %.6g want %.6g (bound %.3g)" % (tuple(i), out[tuple(i)].item(), ref[tuple(i)].item(),
                                                                bound[tuple(i)].item()) for i in idx)
        raise AssertionError("%s: %d of %d elements outside the bound; first: %s" % (what, int(bad.sum()), bad.numel(), shown))


def bf16_rounding_risk(y, delta):
    """Bound on |bf16(y') - bf16(y)| for any y' within delta of y (float64): 0 where no rounding midpoint lies within
    delta of y (both round the same way), else one bf16 ulp of |y| + delta plus delta (each rounding moves by at most
    half an ulp of its own binade).

    A reference that rounds an intermediate to bf16 agrees with a kernel whose fp32 value is within delta of y, except
    where the two sit on either side of a midpoint."""
    a = y.abs().clamp_min(2.0 ** -126)
    ulp = torch.exp2(torch.floor(torch.log2(a)) - 7)
    frac = a / ulp - torch.floor(a / ulp)
    near = (frac - 0.5).abs() * ulp <= delta
    ulp_hi = torch.exp2(torch.floor(torch.log2(a + delta)) - 7)
    return torch.where(near, ulp_hi + delta, torch.zeros_like(ulp))


HOEFFDING = 7.5   # sqrt(2 ln(2 / p)) at p = 1e-12 per element


def random_sign_sum_bound(e, w):
    """Bound on |sum_k d_k w_k| per output for errors |d_k| <= e_k of an operand multiplied by weights w drawn
    independently with random signs (e [M, K], w [N, K] -> [M, N]).  The products are then independent and zero-mean,
    and Hoeffding's inequality puts the sum within HOEFFDING * sqrt(sum e_k^2 w_k^2) except with probability 1e-12.
    Used for the bf16 rounding flips of the FF block's intermediates, which a worst-case sum would overstate ~sqrt(K)
    times."""
    return HOEFFDING * torch.sqrt((e * e) @ (w.double() ** 2).T)


SENTINEL = {torch.bfloat16: (torch.int16, 0x7F81), torch.float32: (torch.int32, 0x7F81C3A5)}  # NaN payloads no kernel writes


def guarded(rows, cols, dtype, device, top=2, bottom=3, left=8, right=8):
    """(buffer, view): a [rows, cols] view at (top, left) of a sentinel-filled [top + rows + bottom, left + cols + right]
    buffer, so its row stride is wider than the row and there are sentinels on all four sides."""
    buf = torch.empty(top + rows + bottom, left + cols + right, dtype=dtype, device=device)
    it, pat = SENTINEL[dtype]
    buf.view(it).fill_(pat)
    return buf, buf[top:top + rows, left:left + cols]


def guarded_flat(n, dtype, device, pad=64):
    buf = torch.empty(n + 2 * pad, dtype=dtype, device=device)
    it, pat = SENTINEL[dtype]
    buf.view(it).fill_(pat)
    return buf, buf[pad:pad + n]


def guard_violations(buf, view):
    """Positions of `buf` outside `view` whose sentinel changed (list of index tuples, at most 5) and their count."""
    it, pat = SENTINEL[buf.dtype]
    outside = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    off = view.storage_offset() - buf.storage_offset()
    if buf.dim() == 1:
        outside[off:off + view.numel()] = False
    else:
        ld = buf.stride(0)
        r0, c0 = off // ld, off % ld
        outside[r0:r0 + view.shape[0], c0:c0 + view.shape[1]] = False
    changed = outside & (buf.view(it) != pat)
    return changed.nonzero()[:5].tolist(), int(changed.sum())


def assert_guard(buf, view, what):
    first, n = guard_violations(buf, view)
    assert n == 0, "%s: %d sentinel elements outside the output were overwritten, first at %s" % (what, n, first)


# ------------------------------------------------------------------------------------------ GEMM reference
def act_ref(v, act):
    if act == ACT_GELU:
        return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))
    if act == ACT_RELU:
        return v.clamp_min(0.0)
    if act == ACT_GELU_TANH:
        return 0.5 * v * (1.0 + torch.tanh(0.7978845608028654 * (v + 0.044715 * v ** 3)))
    if act == ACT_SILU:
        return v * torch.sigmoid(v)
    return v


def gemm_ref(a, w, bias=None, gamma=None, res=None, act=ACT_NONE):
    """float64 epi(a @ w^T) and its magnitude (the same computation on absolute values) for elementwise_bound."""
    a64, w64 = a.double(), w.double()
    v, mag = a64 @ w64.T, a64.abs() @ w64.abs().T
    if bias is not None:
        v, mag = v + bias.double(), mag + bias.double().abs()
    if act == ACT_SWIGLU:   # (gate, up) interleaved columns
        return act_ref(v[:, 0::2], ACT_SILU) * v[:, 1::2], mag[:, 0::2] * mag[:, 1::2]
    v = act_ref(v, act)
    if gamma is not None:
        v, mag = v * gamma.double(), mag * gamma.double().abs()
    if res is not None:
        v, mag = v + res.double(), mag + res.double().abs()
    return v, mag


def gemm_tile_width(M, N, sms):
    """The dispatcher's tile-width rule (gemm_wgmma.cu, gemm_bf16, L452-459): fewest waves times (BN + 48), ties to 128."""
    tm = (M + 127) // 128

    def cost(bn):
        tiles = tm * ((N + bn - 1) // bn)
        return (tiles + sms - 1) // sms * (bn + 48)
    return 128 if cost(128) <= cost(64) else 64


def wgrad_splits(M, No, Ko, sms):
    """wgrad_tn_splits (wgrad_tn.cu): one wave of CTAs over the 128 x 128 output tiles, at most one split per 64 rows, <= 64."""
    tiles = ((No + 127) // 128) * ((Ko + 127) // 128)
    blocks = (M + 63) // 64
    return max(1, min(sms // tiles, blocks, 64))


# ------------------------------------------------------------------------------------------ attention decoys
HD = 128
DECOY_UNIT_NATS = 8.0            # one score unit = P raw (q . k) at scale 8 / P
# Key code per head dim: a P-Hadamard row on key % P, a one-hot (value P) on key // P, one parity column (the last).
# hd -> P; hd - P - 1 block columns, so a sequence of up to P (hd - P - 1) keys is exact (480 / 992 / 960 / 4032).
DECOY_P = {48: 32, 64: 32, 80: 64, 128: 64}
_PARITY = 16                     # units: own-sequence keys -16, opposite-parity keys +16, zero rows 0


def decoy_scale(hd=HD):
    return DECOY_UNIT_NATS / DECOY_P[hd]


def decoy_max_keys(hd=HD):
    """Longest key sequence the decoy code keeps exact at this head dim."""
    P = DECOY_P[hd]
    return P * (hd - P - 1)


DECOY_SCALE = decoy_scale(HD)    # 1/8


def _hadamard(n):
    h = torch.ones(1, 1)
    while h.shape[0] < n:
        h = torch.cat((torch.cat((h, h), 1), torch.cat((h, -h), 1)), 0)
    return h


def decoy_candidates(pos, lim):
    """Target candidates of a query row whose diagonal key is `pos` and whose last visible key is `lim`: key 0, the
    diagonal, the key one 64-key tile back, one spread key and the last key of every 64-key tile."""
    return sorted({0, min(pos, lim), min(max(pos - 64, 0), lim), (pos * 5 + 3) % (lim + 1)} | set(range(63, lim + 1, 64)))


def decoy_key_code(n, sigma, hd=HD):
    """[n, hd] key code of keys 0 .. n - 1 of one sequence with parity sigma (+-1)."""
    P = DECOY_P[hd]
    assert n <= decoy_max_keys(hd), "sequence of %d keys is past the exact decoy limit at hd %d" % (n, hd)
    j = torch.arange(n)
    code = torch.zeros(n, hd)
    code[:, :P] = _hadamard(P)[j % P]
    code[j, P + j // P] = float(P)
    code[:, hd - 1] = -float(P) * sigma
    return code


def decoy_query_code(sq, sk, causal, sigma, hq, hd=HD):
    """Query code of a sequence of sq query rows over sk keys (bottom-right causal: row i sees keys j <= i + sk - sq, so a
    chunk at offset ctx into its keys is sq = n, sk = ctx + n) -> (q [sq, hq, hd], target key per (row, head) [sq, hq]).

    In score units (own-sequence key j scores A[j % P] + B[j // P] - 16): non-causal, the target 6 and every other key
    <= 3.  Causal, the target 12 and every visible key <= 9; where the row can take one, an in-block decoy at key i + 1
    scores 15, and every key of a later P-key block scores >= 15.  Keys of the opposite parity score >= +16 and zero rows
    0.  So the target beats every visible key by >= 3 units (24 nats), and those decoys beat the target by >= 3 units.
    Targets rotate over the candidates by row and head, so each head of a GQA group sees others."""
    P = DECOY_P[hd]
    nb = hd - P - 1
    assert sk <= decoy_max_keys(hd) and (not causal or sq <= sk)
    pos = np.arange(sq) + (sk - sq if causal else 0)
    lim = pos if causal else np.full(sq, sk - 1)
    heads = np.arange(hq)
    # decoy_candidates for every row at once: sorted, duplicates pushed to the end, then picked by (pos * 3 + head)
    big = np.iinfo(np.int64).max
    ends = 63 + 64 * np.arange(max(int(lim.max()) + 1, 0) // 64)
    c = np.concatenate((np.stack((np.zeros(sq, np.int64), np.minimum(pos, lim), np.minimum(np.maximum(pos - 64, 0), lim),
                                  (pos * 5 + 3) % (lim + 1)), 1),
                        np.where(ends[None, :] <= lim[:, None], ends[None, :], big)), 1)
    c.sort(1)
    c[:, 1:][c[:, 1:] == c[:, :-1]] = big
    c.sort(1)
    count = (c != big).sum(1)
    t = np.take_along_axis(c, (pos[:, None] * 3 + heads[None, :]) % count[:, None], 1)
    A = np.zeros((sq, hq, P), dtype=np.float32)
    B = np.zeros((sq, hq, nb), dtype=np.float32)
    r, h = np.arange(sq)[:, None], heads[None, :]
    ta, tb = t % P, t // P
    if not causal:
        A[r, h, ta], B[r, h, tb] = 3, 3
    else:
        ia, ib = np.broadcast_to((pos % P)[:, None], t.shape), np.broadcast_to((pos // P)[:, None], t.shape)
        decoy = np.broadcast_to(((pos + 1 < sk) & (pos % P < P - 1))[:, None], t.shape)
        same = tb == ib
        A[r, h, ta] = np.where(same, 3, 9)
        B[r, h, tb] = np.where(same, 9, 3)
        d = decoy & (same | (ta > ia + 1))   # other block: key (ta, ib) is then hidden too, and A[ia + 1] not the target's
        rr, hh = np.nonzero(d)
        A[rr, hh, ia[rr, hh] + 1] = 6
        B[rr, hh, ib[rr, hh]] = 9
        later = (np.arange(nb)[None, None, :] > ib[:, :, None]) & (np.arange(nb)[None, None, :] < (sk + P - 1) // P)
        B[later] = 15
    q = torch.zeros(sq, hq, hd)
    q[:, :, :P] = torch.from_numpy(A) @ _hadamard(P)
    q[:, :, P:P + nb] = torch.from_numpy(B)
    q[:, :, hd - 1] = _PARITY * sigma
    return q, torch.from_numpy(t)


def decoy_values(rows, cols, gen):
    """V entries: integers of magnitude 1 .. 8 with random signs."""
    return small_ints((rows, cols), 1, 8, gen, torch.float32) * (small_ints((rows, cols), 0, 1, gen, torch.float32) * 2 - 1)


def decoy_expect(v, key_rows, group, hd=HD):
    """Expected output [rows, hq * hd]: row r of head h is V[key_rows[r, h]] of K-V head h // group."""
    hq = key_rows.shape[1]
    kv_cols = (torch.arange(hq) // group)[:, None] * hd + torch.arange(hd)[None, :]
    return v.cpu()[key_rows[:, :, None], kv_cols[None, :, :]].reshape(key_rows.shape[0], hq * hd)


def make_decoy_attention(lens, hkv, group, causal, seed=0, device="cpu", tail_rows=320, hd=HD):
    """Packed var-len decoys: q, k, v bf16 buffers of sum(query lengths) / sum(key lengths) + tail_rows rows (the rows
    past the end hold decoys the kernel must never load) and the expected output: row i of head h is exactly
    V[target(i, h)] of the head's K-V head.  An entry of `lens` is n (n queries over n keys) or (sq, sk).
    Consecutive sequences alternate parity.  -> (q, k, v, expect, targets as rows of k)."""
    hq_total = hkv * group
    P = DECOY_P[hd]
    pairs = [(n, n) if isinstance(n, int) else tuple(n) for n in lens]
    Tq, Tk = sum(sq for sq, _ in pairs), sum(sk for _, sk in pairs)
    gen = torch.Generator().manual_seed(seed)
    q = torch.zeros(Tq + tail_rows, hq_total, hd)
    k = torch.zeros(Tk + tail_rows, hkv, hd)
    v = decoy_values(Tk + tail_rows, hkv * hd, gen)
    targets = torch.zeros(Tq, hq_total, dtype=torch.int64)
    qs = ks = 0
    for b, (sq, sk) in enumerate(pairs):
        sigma = 1 if b % 2 == 0 else -1
        k[ks:ks + sk] = decoy_key_code(sk, sigma, hd)[:, None, :]
        q[qs:qs + sq], t = decoy_query_code(sq, sk, causal, sigma, hq_total, hd)
        targets[qs:qs + sq] = ks + t
        qs, ks = qs + sq, ks + sk
    # rows past the end: every block code and no parity, so they beat any target if they were ever loaded
    k[Tk:, :, P:hd - 1] = float(P)
    q, k, v = (x.reshape(x.shape[0], -1).to(torch.bfloat16).to(device) for x in (q, k, v))
    return q, k, v, decoy_expect(v, targets, group, hd).to(device), targets


def attention_ref_rows(q, k, v, seqs, hkv, group, scale, hd=HD, head_map=None):
    """float64 attention sequence by sequence: seqs = [(q_rows [n], k_rows [m], vis [n])] with q_rows rows of q,
    k_rows rows of k / v (-1: a zero row) and keys [0, vis[i]) of k_rows visible to query row i; GQA head h on K-V head
    head_map(h) (default h // group).  -> (out, mag = sum p |v| / sum p, dlogit = bound on the fp32 logit error (nats)),
    each over the concatenated q_rows."""
    hq_total = hkv * group
    dev = q.device
    heads = torch.arange(hq_total)
    kvh = (head_map(heads) if head_map is not None else heads // group).to(dev)
    zero = lambda x: torch.cat((x.double(), torch.zeros(1, x.shape[1], dtype=torch.float64, device=dev)))
    k64 = zero(k).view(-1, k.shape[1] // hd, hd)[:, :hkv]
    v64 = zero(v).view(-1, v.shape[1] // hd, hd)[:, :hkv]
    outs, mags, dls = [], [], []
    for q_rows, k_rows, vis in seqs:
        q_rows, k_rows, vis = (torch.as_tensor(x, dtype=torch.int64, device=dev) for x in (q_rows, k_rows, vis))
        n, m = q_rows.numel(), k_rows.numel()
        k_rows = torch.where(k_rows < 0, torch.full_like(k_rows, k64.shape[0] - 1), k_rows)
        qs = q[q_rows].double().view(n, -1, hd)[:, :hq_total].transpose(0, 1)              # [hq, n, hd]
        kw = k64[k_rows][:, kvh].transpose(0, 1)                                            # [hq, m, hd]
        vw = v64[k_rows][:, kvh].transpose(0, 1)
        j = torch.arange(m, device=dev)[None, :]
        hide = j >= vis[:, None]
        s = (qs @ kw.transpose(1, 2) * scale).masked_fill(hide, float("-inf"))
        sabs = (qs.abs() @ kw.abs().transpose(1, 2) * scale).masked_fill(hide, 0.0)
        p = torch.softmax(s, -1)
        outs.append((p @ vw).transpose(0, 1).reshape(n, -1))
        mags.append((p @ vw.abs()).transpose(0, 1).reshape(n, -1))
        # fp32 Q K^T over hd products, then s * scale * log2(e) - m * scale * log2(e) and ex2.approx (2 ulp)
        sl = s.masked_fill(hide, 0.0).abs()
        d = (hd + 8) * U32 * sabs.amax(-1) + 8 * U32 * sl.amax(-1) * math.log2(math.e) + 4 * U32
        dls.append(d.transpose(0, 1))
    return torch.cat(outs), torch.cat(mags), torch.cat(dls)


def attention_ref(q, k, v, lens, hkv, group, causal, scale, shift=0, window=320, hd=HD):
    """float64 attention over what the wgmma kernel loads: for each sequence the `window` rows from its start (rows past
    the tensor read as zeros, as TMA fills them), keys [0, visible + shift) of it, GQA head h on K-V head h // group.
    -> (out [T, Hq * hd], mag [T, Hq * hd] = sum p |v| / sum p, dlogit [T, Hq] = bound on the fp32 logit error (nats))."""
    T = sum(lens)
    dev = q.device
    seqs, start = [], 0
    for n in lens:
        i = torch.arange(n, device=dev)
        rows = start + torch.arange(window, device=dev)
        vis = (torch.minimum(i + 1, torch.tensor(n, device=dev)) if causal else torch.full_like(i, n)) + shift
        seqs.append((start + i, torch.where(rows < T, rows, torch.full_like(rows, -1)), vis))
        start += n
    return attention_ref_rows(q[:T], k[:T], v[:T], seqs, hkv, group, scale, hd)


def attention_bound(out_ref, mag, dlogit, group_heads, hd=HD, keys=320):
    """elementwise_bound for the attention output over `keys` keys: P is rounded to bf16 before P V (2^-8 of each p in
    the numerator but not in the row sum), and a logit error d moves each p by a factor within e^{+-d} in numerator and
    denominator."""
    rel = BF16_U + 2.0 * dlogit.repeat_interleave(hd, dim=1)
    return elementwise_bound(out_ref, mag, keys, extra=rel * mag)


def identify_key(row, v, start, kh, window=320, hd=HD, rows=None):
    """Which loaded key's V row (of K-V head kh) the output row equals: for failure messages.  The candidates are the
    `window` rows from `start`, or the given `rows` of v (a sequence's keys, in order)."""
    T = v.shape[0]
    if rows is None:
        rows = torch.arange(start, min(start + window, T))
    cand = v[torch.as_tensor(rows, device=v.device), kh * hd:(kh + 1) * hd].float()
    hit = (cand == row.float()[None, :]).all(1).nonzero()
    if hit.numel():
        return "key %d of the load window (row %d)" % (int(hit[0]), int(rows[int(hit[0])]))
    if bool((row.float() == 0).all()):
        return "a zero row (past the end of the tensor)"
    if bool(torch.isnan(row.float()).any()):
        return "NaN (a row the kernel must not read)"
    return "no single key (a mixture)"


# ------------------------------------------------------------------------------------------ device plumbing
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def L():
    from internnav_b200 import _lib
    _lib.lib()
    return _lib


def _gemm_into(L, a, w, out, bias=None, gamma=None, res=None, act=ACT_NONE):
    """n1_op_gemm into a caller-owned (possibly strided or misaligned) output view."""
    import ctypes
    vp = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    L.check(L.lib().n1_op_gemm(vp(a), a.stride(0), vp(w), w.stride(0), vp(out), out.stride(0), a.shape[0], w.shape[0],
                               a.shape[1], vp(bias), vp(gamma), vp(res), res.stride(0) if res is not None else 0, act,
                               1 if out.dtype == torch.float32 else 0, L.stream_ptr()))


def _attention_into(L, q, k, v, o, cu, max_seq, total_rows, hq, hkv, causal, scale):
    import ctypes
    used = ctypes.c_int(-1)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    L.check(L.lib().n1_op_attention_ex(vp(q), vp(k), vp(v), vp(o), q.stride(0), k.stride(0), v.stride(0), o.stride(0), hq,
                                       hkv, HD, cu.numel() - 1, vp(cu), int(max_seq), int(total_rows), 1 if causal else 0,
                                       float(scale), ctypes.byref(used), L.stream_ptr()))
    return bool(used.value)


# ------------------------------------------------------------------------------------------ GEMM
# (id, shape as a function of the SM count): M % 128 in {1, 63, 64, 65, 127}, N % 32 in {8, 16, 24}, K % 64 in {8, 56}
# and K = 8, both tile widths, tile counts of SM + 1 and 2 SM + 1 (the ring's phase carries from tile to tile inside a
# CTA), and a W over 32 MB whose 20 M tiles are not a multiple of its 18-tile raster group.
GEMM_SHAPES = [
    ("m1_n8_k8", lambda s: (129, 264, 72)),
    ("m63_n16_k56", lambda s: (191, 48, 120)),
    ("m64_n24_k8only", lambda s: (192, 56, 8)),
    ("m65_n8_k8", lambda s: (193, 392, 584)),
    ("m127_n16_k56", lambda s: (255, 1040, 376)),
    ("one_row", lambda s: (1, 24, 56)),
    ("bn128_one_wave", lambda s: ((s // 2 + 1) * 128 - 63, 128, 120)),
    ("tiles_sm_plus_1", lambda s: (s * 128 + 1, 64, 248)),
    ("tiles_2sm_plus_1", lambda s: (2 * s * 128 + 127, 128, 200)),
    ("w_over_32mb", lambda s: (2500, 4736, 3584)),
]


def test_gemm_shape_set_covers_both_tile_widths():
    sms = _sms()
    widths = {gemm_tile_width(*f(sms)[:2], sms) for _, f in GEMM_SHAPES}
    assert widths == {64, 128}, widths
    tiles = {name: ((f(sms)[0] + 127) // 128) * ((f(sms)[1] + gemm_tile_width(*f(sms)[:2], sms) - 1)
                                                // gemm_tile_width(*f(sms)[:2], sms)) for name, f in GEMM_SHAPES}
    assert tiles["tiles_sm_plus_1"] == sms + 1 and tiles["tiles_2sm_plus_1"] == 2 * sms + 1
    M, N, K = dict(GEMM_SHAPES)["w_over_32mb"](sms)
    group = max(2, (16 << 20) // (128 * K * 2))
    assert N * K * 2 > (32 << 20) and ((M + 127) // 128) % group != 0


@pytest.mark.parametrize("name,shape", GEMM_SHAPES, ids=[n for n, _ in GEMM_SHAPES])
def test_gemm_exact_shapes(L, name, shape):
    """Integer operands in [-2, 2], integer bias / gamma / residual: bit-exact against float64, TMA-store epilogue."""
    M, N, K = shape(_sms())
    gen = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a = small_ints((M, K), -2, 2, gen, device="cuda")
    w = small_ints((N, K), -2, 2, gen, device="cuda")
    bias = small_ints((N,), -8, 8, gen, torch.float32, "cuda")
    gamma = small_ints((N,), -2, 2, gen, torch.float32, "cuda")
    res = small_ints((M, N), -64, 64, gen, device="cuda")
    ref, _ = gemm_ref(a, w, bias, gamma, res)
    outs = []
    for _ in range(2):
        buf, out = guarded(M, N, torch.bfloat16, "cuda")
        _gemm_into(L, a, w, out, bias, gamma, res)
        torch.cuda.synchronize()
        assert_guard(buf, out, name)
        outs.append(out.clone())
    assert_exact(outs[0], ref, "%s M=%d N=%d K=%d" % (name, M, N, K))
    assert torch.equal(outs[0], outs[1]), "second call differs"


EPILOGUES = [(), ("bias",), ("gamma",), ("res",), ("bias", "gamma", "res")]


@pytest.mark.parametrize("act,mode", [(act, mode) for act in (ACT_NONE, ACT_GELU, ACT_RELU, ACT_SWIGLU, ACT_GELU_TANH, ACT_SILU)
                                      for mode in ("bf16", "fp32", "inplace") if act != ACT_SWIGLU or mode == "bf16"])
def test_gemm_epilogues(L, act, mode):
    """Every activation x {bias, gamma, residual} x {bf16 out, fp32 out, bf16 in place on the residual}.  M % 128 = 65,
    N % 32 = 16 (SwiGLU's half tile), K % 64 = 56.  Identity and ReLU are bit-exact; GELU, tanh-GELU, SiLU and SwiGLU
    are held to elementwise_bound.  SwiGLU's epilogue takes only the bias and writes bf16."""
    M, N, K = 193, 272, 120
    gen = torch.Generator().manual_seed(act * 10 + len(mode))
    a = small_ints((M, K), -2, 2, gen, device="cuda")
    w = small_ints((N, K), -1, 1, gen, device="cuda")
    n_out = N // 2 if act == ACT_SWIGLU else N
    full = {"bias": small_ints((N,), -6, 6, gen, torch.float32, "cuda"),
            "gamma": small_ints((n_out,), -2, 2, gen, torch.float32, "cuda"),
            "res": small_ints((M, n_out), -32, 32, gen, device="cuda")}
    dtype = torch.float32 if mode == "fp32" else torch.bfloat16
    exact = act in (ACT_NONE, ACT_RELU)
    for epi in EPILOGUES:
        if act == ACT_SWIGLU and epi not in ((), ("bias",)):
            continue
        if mode == "inplace" and "res" not in epi:
            continue
        kw = {e: full[e] for e in epi}
        ref, mag = gemm_ref(a, w, kw.get("bias"), kw.get("gamma"), kw.get("res"), act)
        what = "act=%d %s epilogue=%s" % (act, mode, "+".join(epi) or "none")
        outs = []
        for _ in range(2):
            buf, out = guarded(M, n_out, dtype, "cuda")
            res = kw.get("res")
            if mode == "inplace":
                out.copy_(res)
                res = out
            _gemm_into(L, a, w, out, kw.get("bias"), kw.get("gamma"), res, act)
            torch.cuda.synchronize()
            assert_guard(buf, out, what)
            outs.append(out.clone())
        if exact:
            assert_exact(outs[0], ref, what)
        else:
            assert_within(outs[0], ref, elementwise_bound(ref, mag, K, bf16_out=dtype == torch.bfloat16), what)
        assert torch.equal(outs[0], outs[1]), what + ": second call differs"


@pytest.mark.parametrize("layout", ["offset_8_bytes", "ldo_mod_8_is_2"])
@pytest.mark.parametrize("act", [ACT_NONE, ACT_SWIGLU])
def test_gemm_direct_store(L, act, layout):
    """An output that is 8 but not 16 bytes aligned, or whose row stride is not a multiple of 8, cannot be a TMA store
    target: the epilogue stores from registers instead.  Bit-exact (plain) or bounded (SwiGLU), guard band intact."""
    M, N, K = 255, 272, 184
    gen = torch.Generator().manual_seed(act + len(layout))
    a = small_ints((M, K), -2, 2, gen, device="cuda")
    w = small_ints((N, K), -1, 1, gen, device="cuda")
    n_out = N // 2 if act == ACT_SWIGLU else N
    bias = small_ints((N,), -6, 6, gen, torch.float32, "cuda")
    gamma = None if act == ACT_SWIGLU else small_ints((N,), -2, 2, gen, torch.float32, "cuda")
    res = None if act == ACT_SWIGLU else small_ints((M, N), -32, 32, gen, device="cuda")
    left, right = (4, 4) if layout == "offset_8_bytes" else (8, 10)
    buf, out = guarded(M, n_out, torch.bfloat16, "cuda", left=left, right=right)
    assert out.data_ptr() % 16 != 0 or out.stride(0) % 8 != 0
    _gemm_into(L, a, w, out, bias, gamma, res, act)
    torch.cuda.synchronize()
    assert_guard(buf, out, layout)
    ref, mag = gemm_ref(a, w, bias, gamma, res, act)
    if act == ACT_SWIGLU:
        assert_within(out, ref, elementwise_bound(ref, mag, K), layout)
    else:
        assert_exact(out, ref, layout)


# ------------------------------------------------------------------------------------------ weight gradient
WGRAD_CASES = [
    ("last_split_empty", lambda s: (65 * 64 - 5, 128, 128)),
    ("tails_no8_ko72", lambda s: (1000, 136, 200)),
    ("m_below_64", lambda s: (37, 264, 136)),
    ("m_mod64_is_1_multi_tile", lambda s: (577, 384, 1160)),
]


@pytest.mark.parametrize("name,shape", WGRAD_CASES, ids=[n for n, _ in WGRAD_CASES])
def test_wgrad_exact(name, shape):
    """dW = dY^T X on integer operands in [-2, 2]: bit-exact against float64, written and accumulated onto an integer
    target, with sentinels on both sides of the output."""
    from internnav_b200 import _bwd as K
    sms = _sms()
    M, No, Ko = shape(sms)
    if name == "last_split_empty":
        sp = wgrad_splits(M, No, Ko, sms)
        per = -(-((M + 63) // 64) // sp)
        assert (sp - 1) * per >= (M + 63) // 64, "the last split should get no rows"
    gen = torch.Generator().manual_seed(M + No + Ko)
    dy = small_ints((M, No), -2, 2, gen, device="cuda")
    x = small_ints((M, Ko), -2, 2, gen, device="cuda")
    ref = dy.double().T @ x.double()
    init = small_ints((No, Ko), -50, 50, gen, torch.float32, "cuda")
    outs = []
    for accumulate in (False, True, False):
        buf, flat = guarded_flat(No * Ko, torch.float32, "cuda")
        out = flat.view(No, Ko)
        if accumulate:
            out.copy_(init)
        K.wgrad(dy, x, out=out, accumulate=accumulate)
        torch.cuda.synchronize()
        assert_guard(buf, flat, "%s accumulate=%s" % (name, accumulate))
        assert_exact(out, ref + (init.double() if accumulate else 0), "%s accumulate=%s" % (name, accumulate))
        outs.append(out.clone())
    assert torch.equal(outs[0], outs[2]), "second call differs"


# ------------------------------------------------------------------------------------------ wgmma attention
def _run_decoys(L, lens, hkv, group, causal, seed=0, expect_tc=True):
    q, k, v, expect, targets = make_decoy_attention(lens, hkv, group, causal, seed=seed, device="cuda")
    T, hq = sum(lens), hkv * group
    cu = torch.tensor([0] + [sum(lens[:i + 1]) for i in range(len(lens))], dtype=torch.int32, device="cuda")
    outs = []
    for _ in range(2):
        buf, o = guarded(T, hq * HD, torch.bfloat16, "cuda", top=1, bottom=4, left=64, right=72)
        used = _attention_into(L, q[:T], k[:T], v[:T], o, cu, max(lens), T, hq, hkv, causal, DECOY_SCALE)
        torch.cuda.synchronize()
        assert used == expect_tc, "wgmma kernel %s, expected %s" % ("ran" if used else "did not run", expect_tc)
        assert_guard(buf, o, "attention output")
        outs.append(o.clone())
    o = outs[0]
    bad = (o.view(torch.int16) != expect.view(torch.int16)).view(T, hq, HD).any(-1)
    if bool(bad.any()):
        r, h = (int(x) for x in bad.nonzero()[0])
        b = int((cu[1:].cpu() <= r).sum())
        start = int(cu[b])
        saw = identify_key(o[r, h * HD:(h + 1) * HD], v, start, h // group)
        raise AssertionError("%d of %d (row, head) outputs wrong; first: sequence %d (len %d) row %d head %d should see "
                             "key %d only, saw %s" % (int(bad.sum()), bad.numel(), b, lens[b], r - start, h,
                                                      int(targets[r, h]) - start, saw))
    assert torch.equal(outs[0], outs[1]), "second call differs"


ATTN_LENGTHS = [1, 63, 64, 65, 127, 128, 129, 191, 192, 255, 256, 257, 319, 320]


@pytest.mark.parametrize("group", [1, 2, 7])
@pytest.mark.parametrize("causal", [True, False])
def test_attention_decoys_every_length(L, causal, group):
    """Every 64 / 128 boundary of the sequence length in one packed batch (each sequence followed by the next one
    inside its 320-row load, the last one by the end of the tensor); every output row must be exactly its target's V."""
    _run_decoys(L, ATTN_LENGTHS, 2, group, causal, seed=group)


def test_attention_decoys_two_uneven_waves(L):
    """64 x 304 tokens, 28 / 4 heads: 256 work items over the SMs, a second wave on part of them; every sequence,
    head and row checked."""
    _run_decoys(L, [304] * 64, 4, 7, True, seed=5)


def test_attention_decoys_321_takes_mma_sync(L):
    """A 321-token sequence is past the wgmma kernel's 320-key load: the call must report the mma.sync kernel and pass
    the same checks."""
    _run_decoys(L, [321, 64, 200], 2, 2, True, seed=7, expect_tc=False)


@pytest.mark.parametrize("causal", [True, False])
def test_attention_softmax_rescaling(L, causal):
    """Random data with logits up to ~60 nats whose row maximum rises from key block to key block (the last visible
    block holds it), a non-default scale, and the output in a wider row-stride buffer with a guard band; every element
    against the float64 softmax with attention_bound."""
    lens = [1, 65, 129, 200, 257, 320]
    hkv, group = 2, 7
    hq, T = hkv * group, sum(lens)
    scale = 0.0625
    gen = torch.Generator().manual_seed(11 + causal)
    q = torch.randn(T, hq * HD, generator=gen)
    k = torch.randn(T, hkv * HD, generator=gen) * 1.5
    v = torch.randn(T, hkv * HD, generator=gen)
    q.view(T, hq, HD)[:, :, 0] = 8.0
    start = 0
    for n in lens:   # dim 0 of the keys: a ramp to 60 nats (8 * 120 * 0.0625) at the sequence's last key
        k.view(T, hkv, HD)[start:start + n, :, 0] = (120.0 * (torch.arange(n) + 1) / n)[:, None]
        start += n
    q, k, v = (x.bfloat16().cuda() for x in (q, k, v))
    cu = torch.tensor([0] + [sum(lens[:i + 1]) for i in range(len(lens))], dtype=torch.int32, device="cuda")
    buf, o = guarded(T, hq * HD, torch.bfloat16, "cuda", top=1, bottom=4, left=64, right=72)
    assert _attention_into(L, q, k, v, o, cu, max(lens), T, hq, hkv, causal, scale)
    torch.cuda.synchronize()
    assert_guard(buf, o, "attention output")
    ref, mag, dl = attention_ref(q, k, v, lens, hkv, group, causal, scale)
    assert float(dl.max()) < 1e-3
    assert_within(o, ref, attention_bound(ref, mag, dl, group), "softmax rescaling causal=%s" % causal)


_CHILD = r"""
import json, sys, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2])
import test_hopper_kernels_gpu as H
from internnav_b200 import _lib as L
lens = [129, 64]
q, k, v, expect, _ = H.make_decoy_attention(lens, 2, 2, True, seed=3, device="cuda")
T = sum(lens)
cu = torch.tensor([0, 129, T], dtype=torch.int32, device="cuda")
o, used = L.attention_varlen(q[:T], k[:T], v[:T], 4, 2, 128, cu, max(lens), causal=True, scale=H.DECOY_SCALE)
torch.cuda.synchronize()
print(json.dumps({"used": used, "exact": bool(torch.equal(o.view(torch.int16), expect.view(torch.int16)))}))
"""


def test_attention_tc_disabled_by_environment_reports_mma_sync():
    """N1_ATTN_TC=0 routes a wgmma-eligible call to the mma.sync kernel, and the call must say so."""
    env = dict(os.environ, N1_ATTN_TC="0")
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, os.path.dirname(os.path.abspath(__file__))], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert got == {"used": False, "exact": True}, got


# ------------------------------------------------------------------------------------------ FF block
D, F = 384, 1536


def ff_ref(x, lw, lb, w1, b1, w2, b2, eps):
    """float64 FF block with the kernel's two bf16 roundings (LayerNorm output, GELU hidden) -> (out, bound).

    Where the kernel's fp32 intermediate may round to the other side of a bf16 midpoint than the float64 one, the two
    differ by about one ulp (bf16_rounding_risk); those ulps are carried through the GEMMs, whose weights have random
    signs, into the bound's `extra` term (random_sign_sum_bound)."""
    x64 = x.double()
    mu = x64.mean(-1, keepdim=True)
    xc = x64 - mu
    var = (xc * xc).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    hn = xc * rstd * lw.double() + lb.double()
    # fp32 LayerNorm error: the mean's sum is exact when every x is a multiple of the row's smallest ulp and the sum
    # stays below 2^24 of them, else (D - 1) 2^-24 sum |x| (Higham 3.5); the variance of the shifted values picks up
    # e_mu^2 plus (D + 16) units; rsqrtf adds 2 ulp
    ax = x64.abs()
    q = torch.exp2(torch.floor(torch.log2(ax.clamp_min(2.0 ** -126))) - 7).amin(-1, keepdim=True)
    exact_sum = (ax.sum(-1, keepdim=True) / q) < 2.0 ** 24
    e_mu = torch.where(exact_sum, 2 * U32 * mu.abs(), (D + 8) * U32 * ax.mean(-1, keepdim=True))
    e_rstd = 0.5 * ((D + 16) * U32 * var + e_mu ** 2) / (var + eps) + 4 * U32
    d_h = lw.double().abs() * rstd * (e_mu + xc.abs() * e_rstd) + 4 * U32 * (hn.abs() + lb.double().abs())
    h = hn.to(torch.bfloat16).double()
    e_h = bf16_rounding_risk(hn, d_h)
    w1a, w2a = w1.double().abs(), w2.double().abs()
    pre = h @ w1.double().T + b1.double()
    m_pre = h.abs() @ w1a.T + b1.double().abs()
    e_pre = (D + 64) * U32 * m_pre + random_sign_sum_bound(e_h, w1)
    g = act_ref(pre, ACT_GELU)
    hid = g.to(torch.bfloat16).double()
    e_hid = bf16_rounding_risk(g, 1.13 * e_pre + 64 * U32 * pre.abs())
    out = x64 + hid @ w2.double().T + b2.double()
    mag = x64.abs() + hid.abs() @ w2a.T + b2.double().abs()
    return out, elementwise_bound(out, mag, F, extra=random_sign_sum_bound(e_hid, w2))


def _ff_operands(M, seed):
    """Rows of three kinds: x ~ 100 + N(0, 1) (the two-pass variance must cancel the mean), N(0.3, 1.5^2), and
    N(0, 2^-18) whose variance is near eps, so that eps = 1e-6 against 1e-5 matters."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(M, D, generator=gen)
    kind = torch.arange(M) % 3
    x[kind == 0] += 100.0
    x[kind == 1] = x[kind == 1] * 1.5 + 0.3
    x[kind == 2] *= 2.0 ** -9
    w1 = (torch.randn(F, D, generator=gen) / math.sqrt(D)).bfloat16()
    w2 = (torch.randn(D, F, generator=gen) / math.sqrt(F)).bfloat16()
    b1, b2 = torch.randn(F, generator=gen) * 0.1, torch.randn(D, generator=gen) * 0.1
    lw, lb = 1 + 0.1 * torch.randn(D, generator=gen), 0.1 * torch.randn(D, generator=gen)
    return [t.cuda() for t in (x.bfloat16(), lw, lb, w1, b1, w2, b2)]


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("M", [1, 63, 64, 65, 129, 192])
def test_ff_block_tile_edges(L, M, seed):
    """M below, at and past the 64-row tile, x and out as column slices of wider buffers with sentinels around them, then
    in place; eps = 1e-6."""
    x, lw, lb, w1, b1, w2, b2 = _ff_operands(M, M * 2 + seed)
    eps = 1e-6
    ref, bound = ff_ref(x, lw, lb, w1, b1, w2, b2, eps)
    xbuf, xv = guarded(M, D, torch.bfloat16, "cuda", left=16, right=24)
    xv.copy_(x)
    xsnap = xbuf.clone()
    outs = []
    for _ in range(2):
        obuf, ov = guarded(M, D, torch.bfloat16, "cuda", left=8, right=40)
        L.ff_block(xv, lw, lb, w1, b1, w2, b2, eps=eps, out=ov)
        torch.cuda.synchronize()
        assert_guard(obuf, ov, "ff_block out")
        assert torch.equal(xbuf.view(torch.int16), xsnap.view(torch.int16)), "ff_block wrote into its input"
        outs.append(ov.clone())
    assert_within(outs[0], ref, bound, "ff_block M=%d seed=%d" % (M, seed))
    assert torch.equal(outs[0], outs[1]), "second call differs"
    # in place on the residual stream slice, as the decoder runs it
    L.ff_block(xv, lw, lb, w1, b1, w2, b2, eps=eps, out=xv)
    torch.cuda.synchronize()
    assert_guard(xbuf, xv, "ff_block in place")
    assert torch.equal(xv, outs[0]), "in-place result differs"
