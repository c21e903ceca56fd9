"""The checks of tests/test_hopper_kernels_gpu.py, run on the CPU against float64 references that carry the errors those
tests exist to catch: each must be rejected, and the correct result accepted.  Also checks that the attention decoy
construction separates every target from what its row may and may not see by more than 20 nats."""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_hopper_kernels_gpu as H  # noqa: E402


def _ints(shape, lo, hi, seed):
    return H.small_ints(shape, lo, hi, torch.Generator().manual_seed(seed))


def _drop_kstep(a, w, ref, rows, cols, k0):
    """ref with one 16-wide k-step (k0 .. k0 + 15) missing from one output tile"""
    bad = ref.clone()
    bad[rows, cols] -= a[rows, k0:k0 + 16].double() @ w[cols, k0:k0 + 16].double().T
    return bad


def test_exact_check_rejects_a_dropped_kstep_and_accepts_the_result():
    M, N, K = 300, 200, 120
    a, w = _ints((M, K), -2, 2, 1), _ints((N, K), -2, 2, 2)
    res = _ints((M, N), -64, 64, 3)
    ref, _ = H.gemm_ref(a, w, res=res)
    bad, _ = H.exact_mismatches(ref.to(torch.bfloat16), ref)
    assert not bool(bad.any())
    for rows, cols, k0 in [(slice(256, 300), slice(128, 192), 48), (slice(0, 128), slice(192, 200), 0),
                           (slice(128, 256), slice(0, 64), 112 - 8)]:
        broken = _drop_kstep(a, w, ref, rows, cols, k0).to(torch.bfloat16)
        bad, _ = H.exact_mismatches(broken, ref)
        assert bool(bad[rows, cols].any()) and not bool((bad & ~_mask(bad.shape, rows, cols)).any())


def _mask(shape, rows, cols):
    m = torch.zeros(shape, dtype=torch.bool)
    m[rows, cols] = True
    return m


def test_bound_rejects_a_wrong_tail_tile_and_accepts_the_result():
    """GELU epilogue on integer operands: the correctly rounded result is inside elementwise_bound; the last partial M
    tile computed with one k-step missing, or with the bias of the neighbouring column, is not."""
    M, N, K = 193, 272, 120
    a, w = _ints((M, K), -2, 2, 4), _ints((N, K), -1, 1, 5)
    bias = _ints((N,), -6, 6, 6).float()
    for act in (H.ACT_GELU, H.ACT_GELU_TANH, H.ACT_SILU):
        ref, mag = H.gemm_ref(a, w, bias=bias, act=act)
        bound = H.elementwise_bound(ref, mag, K)
        assert not bool(H.bound_violations(ref.to(torch.bfloat16), ref, bound)[0].any())
        tail = slice(128, M)
        v = a.double() @ w.double().T + bias.double()
        dropped = v.clone()
        dropped[tail, 64:128] -= a[tail, 32:48].double() @ w[64:128, 32:48].double().T
        shifted = v.clone()
        shifted[tail, 64:128] += (bias[65:129] - bias[64:128]).double()
        for wrong in (dropped, shifted):
            bad, _ = H.bound_violations(H.act_ref(wrong, act).to(torch.bfloat16), ref, bound)
            assert bool(bad[tail, 64:128].any()), act


def test_guard_band_reports_a_row_past_m_and_a_column_past_n():
    for dtype in (torch.bfloat16, torch.float32):
        buf, view = H.guarded(10, 16, dtype, "cpu")
        view.fill_(1.0)
        assert H.guard_violations(buf, view)[1] == 0
        past_m = buf.clone()
        past_m[2 + 10, 8:24] = 1.0   # row M: the first row below the output
        first, n = H.guard_violations(past_m, past_m[2:12, 8:24])
        assert n == 16 and first[0] == [12, 8]
        past_n = buf.clone()
        past_n[5, 8 + 16] = 2.0      # column N of one row
        assert H.guard_violations(past_n, past_n[2:12, 8:24])[1] == 1
        before = buf.clone()
        before[2, 7] = 3.0           # one column left of the slice
        assert H.guard_violations(before, before[2:12, 8:24])[1] == 1
    buf, flat = H.guarded_flat(100, torch.float32, "cpu")
    flat.fill_(0.0)
    assert H.guard_violations(buf, flat)[1] == 0
    buf[64 + 100] = 0.0
    assert H.guard_violations(buf, flat)[1] == 1


LENS = [1, 63, 64, 65, 127, 128, 129, 191, 192, 255, 256, 257, 319, 320]


def _window_scores(q, k, lens, hkv, group, start, n, window=320):
    """float64 scores in nats of one sequence's rows against the 320 rows the kernel loads (zeros past the tensor)"""
    T = sum(lens)
    kk = torch.cat((k[:T].double(), torch.zeros(window, k.shape[1], dtype=torch.float64)))[start:start + window]
    qs = q[start:start + n].double().view(n, hkv * group, H.HD)
    kw = kk.view(window, hkv, H.HD).repeat_interleave(group, 1)
    return torch.einsum("ihd,jhd->ihj", qs, kw) * H.DECOY_SCALE


def test_decoys_put_the_target_20_nats_from_everything_else():
    """For every (row, head): the target beats every other key the row may see by more than 20 nats, and whenever the
    kernel's 320-row load holds keys of the next sequence, zero rows past the tensor, or (causal) keys of a later
    64-key block, the strongest key the row must not see beats the target by more than 20 nats.  For causal rows, key
    i + 1 itself is such a decoy for most rows."""
    for causal in (True, False):
        for group in (1, 7):
            hkv = 2
            q, k, v, expect, targets = H.make_decoy_attention(LENS, hkv, group, causal, seed=group)
            start, shifted_decoys, shiftable = 0, 0, 0
            for n in LENS:
                s = _window_scores(q, k, LENS, hkv, group, start, n)               # [n, hq, 320]
                i = torch.arange(n)[:, None, None]
                j = torch.arange(320)[None, None, :]
                vis = (j <= i) & (j < n) if causal else (j < n).expand(n, 1, 320)
                t = (targets[start:start + n] - start)[:, :, None]
                st = s.gather(2, t)
                others = s.masked_fill(~vis | (j == t), -math.inf).amax(2, keepdim=True)
                assert bool((st - others > 20).all()), (causal, group, n, float((st - others).min()))
                hidden = s.masked_fill(vis.expand_as(s), -math.inf).amax(2, keepdim=True)
                # rows that load a key past their sequence or (causal) a key of a later 64-key block
                has_decoy = ((j >= n) | ((j // 64 > i // 64) & causal)).any(2, keepdim=True).expand_as(st)
                assert bool(((hidden - st > 20) | ~has_decoy).all()), (causal, group, n)
                if causal and n > 1:
                    nxt = s[torch.arange(n - 1), :, torch.arange(1, n)]            # key i + 1 for rows 0 .. n - 2
                    shifted_decoys += int((nxt - st[:-1, :, 0] > 20).sum())
                    shiftable += nxt.numel()
                start += n
            if causal:
                assert shifted_decoys >= 0.4 * shiftable, (shifted_decoys, shiftable)


def test_decoy_reference_is_exact_and_a_shifted_mask_is_caught():
    """The float64 attention over the decoy data rounds to exactly the expected V rows; with the mask shifted by one key
    (each row also sees key i + 1, or key n for the non-causal rows) the exact check fails for the rows that key beats."""
    lens = [130, 70, 64]
    for causal in (True, False):
        q, k, v, expect, _ = H.make_decoy_attention(lens, 1, 2, causal, seed=1)
        out, _, _ = H.attention_ref(q, k, v, lens, 1, 2, causal, H.DECOY_SCALE)
        assert torch.equal(out.to(torch.bfloat16), expect)
        leak, _, _ = H.attention_ref(q, k, v, lens, 1, 2, causal, H.DECOY_SCALE, shift=1)
        wrong = (leak.to(torch.bfloat16) != expect).view(sum(lens), 2, H.HD).any(-1)
        assert float(wrong.float().mean()) > (0.4 if causal else 0.99), float(wrong.float().mean())
