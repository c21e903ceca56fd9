"""Paged K/V pool on the CPU: the page accounting n1_llm_generate runs before it launches (n1_kv_pages_*), the decoy
construction of the paged attention tests (tests/test_kv_pages_gpu.py) with the exact check rejecting references that
address pages wrongly, and the changed kernels compiling for sm_90a without spills."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_hopper_kernels_gpu as H  # noqa: E402

PAGE = 64
N1_ERR_KV_PAGES = -8


# ------------------------------------------------------------------------------------------ page accounting
class Pages:
    """ctypes view of one host page allocator."""

    def __init__(self, slots, max_tokens, pages):
        from internnav_b200 import _lib
        self.L = _lib.lib()
        self.slots, self.per_slot, self.pages = slots, -(-max_tokens // PAGE), pages
        h = ctypes.c_void_p()
        assert self.L.n1_kv_pages_create(slots, max_tokens, pages, ctypes.byref(h)) == 0
        self.h = h

    def __del__(self):
        self.L.n1_kv_pages_destroy(self.h)

    def prepare(self, slots, keep, need):
        a = lambda v: (ctypes.c_int32 * len(v))(*v)
        ch = (ctypes.c_int32 * 2)()
        rc = self.L.n1_kv_pages_prepare(self.h, len(slots), a(slots), a(keep), a(need), ch)
        return rc, (ch[0], ch[1])

    def trim(self, slot, rows):
        assert self.L.n1_kv_pages_trim(self.h, slot, rows) == 0

    def state(self):
        t = (ctypes.c_int32 * (self.slots * self.per_slot))()
        held = (ctypes.c_int32 * self.slots)()
        fr = (ctypes.c_int32 * self.pages)()
        n = self.L.n1_kv_pages_table(self.h, t, held, fr)
        return np.array(t).reshape(self.slots, self.per_slot), list(held), list(fr)[:n]

    def check(self):
        """free + held = total, no page twice, every slot's pages are the first `held` entries of its table row."""
        table, held, free = self.state()
        owned = [int(p) for s in range(self.slots) for p in table[s, :held[s]]]
        assert all((table[s, held[s]:] == -1).all() for s in range(self.slots))
        assert len(owned) + len(free) == self.pages
        assert sorted(owned + free) == list(range(self.pages))   # no page belongs to two slots or to a slot and the list
        return table, held, free


def test_pages_follow_the_conversations():
    a = Pages(slots=4, max_tokens=300, pages=12)
    assert a.check()[1] == [0, 0, 0, 0]
    # two fresh sequences: prompt + budget rows
    rc, ch = a.prepare([1, 3], [0, 0], [150, 70])
    assert rc == 0 and ch == (1, 4)
    table, held, free = a.check()
    assert held == [0, 3, 0, 2]
    # after the call each slot keeps ceil(valid / 64) pages
    a.trim(1, 130), a.trim(3, 64)
    table, held, _ = a.check()
    assert held == [0, 3, 0, 1]
    prefix = table[1, :2].copy()
    # a continued sequence keeps the pages of its reused prefix (rows 0 .. 127 here), the rest is returned and retaken
    rc, _ = a.prepare([1], [128], [128 + 100])
    assert rc == 0
    table, held, _ = a.check()
    assert held[1] == 4 and (table[1, :2] == prefix).all()
    a.trim(1, 200)
    # a fresh sequence on a written slot gives its old pages back before it takes new ones
    old = set(a.state()[0][1, :a.state()[1][1]].tolist())
    free_before = len(a.state()[2])
    rc, _ = a.prepare([1], [0], [60])
    assert rc == 0
    table, held, free = a.check()
    assert held[1] == 1 and len(free) == free_before + len(old) - 1
    assert set(free) >= old - {int(table[1, 0])}


def test_a_refused_request_leaves_the_state_identical():
    a = Pages(slots=3, max_tokens=512, pages=6)
    assert a.prepare([0], [0], [256])[0] == 0
    a.trim(0, 200)
    before = a.check()
    # slot 0 keeps its 4 pages (200 rows) and needs a fifth, slot 2 needs 5: 6 pages from a list of 2 (+ 0 returned)
    rc, _ = a.prepare([0, 2], [200, 0], [300, 320])
    assert rc == N1_ERR_KV_PAGES
    msg = a.L.n1_last_error().decode()
    assert "needs 6 pages" in msg and "2 are free" in msg, msg
    after = a.check()
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    # a sequence beyond the per-slot bound, or a prefix beyond what the slot holds, is an argument error, also unchanged
    assert a.prepare([1], [0], [513])[0] == -2
    assert a.prepare([1], [64], [100])[0] == -2
    assert all(np.array_equal(x, y) for x, y in zip(before, a.check()))


def test_random_operations_keep_the_books():
    rng = np.random.default_rng(0)
    a = Pages(slots=6, max_tokens=640, pages=24)
    valid = [0] * 6
    for _ in range(400):
        if rng.random() < 0.2:
            s = int(rng.integers(6))
            a.trim(s, 0)
            valid[s] = 0
        else:
            slots = sorted(rng.choice(6, size=int(rng.integers(1, 4)), replace=False).tolist())
            keep = [int(rng.integers(0, valid[s] + 1)) for s in slots]
            need = [min(640, k + int(rng.integers(1, 300))) for k in keep]
            before = a.state()
            held0 = {s: before[0][s, :-(-k // PAGE)].copy() for s, k in zip(slots, keep)}
            rc, _ = a.prepare(slots, keep, need)
            table, held, _ = a.check()
            if rc == N1_ERR_KV_PAGES:
                assert all(np.array_equal(x, y) for x, y in zip(before, a.state()))
                continue
            assert rc == 0
            for s, k, n in zip(slots, keep, need):
                assert held[s] == -(-n // PAGE) and (table[s, :len(held0[s])] == held0[s]).all()
                valid[s] = int(rng.integers(k, n + 1))
                a.trim(s, valid[s])
            table, held, _ = a.check()
            assert all(held[s] == -(-valid[s] // PAGE) for s in slots)


# ------------------------------------------------------------------------------------------ paged decoys
def paged_decoys(pairs, hq, hkv, causal, n_pages=None, shuffle=True, seed=0, nan_rest=True, sigma=None):
    """Decoy attention over a paged pool: sequence b = (sq, sk) has its sk keys on ceil(sk / 64) pages taken from a
    (shuffled) list of n_pages pages; its key j lives at row table[b][j // 64] * 64 + j % 64.  Every row no sequence
    owns is NaN (nan_rest).  -> dict(q, k, v bf16, expect, seqs = [(q_rows, k_rows, vis)], tables [B][n] page lists,
    table [B, per] int32 (-1 padded), per)."""
    hd, group = 128, hq // hkv
    gen = torch.Generator().manual_seed(seed)
    need = [-(-sk // PAGE) for _, sk in pairs]
    per = max(need) + 1
    n_pages = n_pages or sum(need) + 3
    order = torch.randperm(n_pages, generator=gen).tolist() if shuffle else list(range(n_pages))
    rows = n_pages * PAGE
    k = torch.full((rows, hkv * hd), float("nan")) if nan_rest else torch.zeros(rows, hkv * hd)
    v = H.decoy_values(rows, hkv * hd, gen)
    owned = torch.zeros(rows, dtype=torch.bool)
    q = torch.zeros(sum(sq for sq, _ in pairs), hq * hd)
    tables, seqs, targets, qs = [], [], [], 0
    table = torch.full((len(pairs), per), -1, dtype=torch.int32)
    for b, (sq, sk) in enumerate(pairs):
        pg, order = order[:need[b]], order[need[b]:]
        tables.append(pg)
        table[b, :len(pg)] = torch.tensor(pg, dtype=torch.int32)
        j = torch.arange(sk)
        k_rows = torch.tensor(pg)[j // PAGE] * PAGE + j % PAGE
        sg = 1 if sigma is None else sigma[b]
        k[k_rows] = H.decoy_key_code(sk, sg, hd).repeat(1, hkv)
        owned[k_rows] = True
        qc, t = H.decoy_query_code(sq, sk, causal, sg, hq, hd)
        q[qs:qs + sq] = qc.reshape(sq, -1)
        targets.append(k_rows[t])
        i = torch.arange(sq)
        seqs.append((qs + i, k_rows, i + sk - sq + 1 if causal else torch.full((sq,), sk)))
        qs += sq
    if nan_rest:
        v[~owned] = float("nan")
    q, k, v = (x.to(torch.bfloat16) for x in (q, k, v))
    expect = H.decoy_expect(v, torch.cat(targets), group, hd)
    return dict(q=q, k=k, v=v, expect=expect, seqs=seqs, tables=tables, table=table, per=per, pairs=pairs)


def _remap(d, f):
    """seqs with key j of sequence b at f(table_b, j) instead of table_b[j // 64] * 64 + j % 64."""
    out = []
    for (qr, kr, vis), pg in zip(d["seqs"], d["tables"]):
        out.append((qr, torch.tensor([f(pg, j) for j in range(kr.numel())]), vis))
    return out


def _page_off(d):   # every key one page further along the slot's table (the last page wraps to the first)
    return _remap(d, lambda pg, j: pg[(j // PAGE + 1) % len(pg)] * PAGE + j % PAGE)


def _boundary_off_by_one(d):   # the last row of each page taken from the next page
    return _remap(d, lambda pg, j: pg[min((j + 1) // PAGE, len(pg) - 1)] * PAGE + j % PAGE)


def _drop_partial_page(d):
    return [(qr, kr, vis.clamp(max=PAGE * (kr.numel() // PAGE))) for qr, kr, vis in d["seqs"]]


PAGED_FORMS = {   # name -> (query / key lengths, causal)
    "decode": ([(1, 63), (1, 64), (1, 65), (1, 127), (1, 128), (1, 129)], True),
    "latent": ([(5, 63), (5, 64), (5, 65), (5, 127), (5, 128), (5, 129)], True),
    "chunk": ([(17, 17 + 64), (64, 64 + 128), (30, 50 + 30), (1, 129), (65, 65), (100, 127 + 100)], True),
}
MUTATIONS = {
    "one_page_off": _page_off,
    "partial_last_page_dropped": _drop_partial_page,
    "page_boundary_off_by_one": _boundary_off_by_one,
}


@pytest.mark.parametrize("form", sorted(PAGED_FORMS))
def test_paged_decoys_reference_is_exact(form):
    pairs, causal = PAGED_FORMS[form]
    d = paged_decoys(pairs, 28, 4, causal)
    out, _, _ = H.attention_ref_rows(d["q"], d["k"], d["v"], d["seqs"], 4, 7, H.decoy_scale(128))
    assert torch.equal(out.to(torch.bfloat16).view(torch.int16), d["expect"].view(torch.int16))


@pytest.mark.parametrize("name", sorted(MUTATIONS))
@pytest.mark.parametrize("form", sorted(PAGED_FORMS))
def test_exact_check_rejects_wrong_page_addressing(form, name):
    pairs, causal = PAGED_FORMS[form]
    d = paged_decoys(pairs, 8, 2, causal, nan_rest=False)   # without NaN: the decoys alone catch it
    bad, _, _ = H.attention_ref_rows(d["q"], d["k"], d["v"], MUTATIONS[name](d), 2, 4, H.decoy_scale(128))
    assert bool((bad.to(torch.bfloat16).view(torch.int16) != d["expect"].view(torch.int16)).any()), name


def stale_page_decoys(hq=8, hkv=2):
    """Sequence 0 (100 keys) once held pages [a, b]; page b went back to the free list and now holds sequence 1's first
    64 keys, while sequence 0 holds [a, c].  -> (decoys, sequence 0's rows through its stale table)."""
    d = paged_decoys([(5, 100), (5, 130)], hq, hkv, True, nan_rest=False, sigma=[1, -1])
    a, c = d["tables"][0]
    b = d["tables"][1][0]
    stale = [a, b]
    j = torch.arange(100)
    rows = torch.tensor(stale)[j // PAGE] * PAGE + j % PAGE
    return d, [(d["seqs"][0][0], rows, d["seqs"][0][2])] + d["seqs"][1:]


def test_exact_check_rejects_a_page_the_slot_no_longer_holds():
    d, wrong = stale_page_decoys()
    good, _, _ = H.attention_ref_rows(d["q"], d["k"], d["v"], d["seqs"], 2, 4, H.decoy_scale(128))
    assert torch.equal(good.to(torch.bfloat16).view(torch.int16), d["expect"].view(torch.int16))
    bad, _, _ = H.attention_ref_rows(d["q"], d["k"], d["v"], wrong, 2, 4, H.decoy_scale(128))
    n0 = d["pairs"][0][0]
    assert bool((bad[:n0].to(torch.bfloat16).view(torch.int16) != d["expect"][:n0].view(torch.int16)).any())


# ------------------------------------------------------------------------------------------ compile
def _nvcc():
    from internnav_b200 import build
    return build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not installed")
@pytest.mark.parametrize("src,kernel,entries", [("attention.cu", "attn_kernel", 5),
                                                ("attention_cache_wgmma.cu", "attn_cache_kernel", 1),
                                                ("s2_kernels.cu", "gen_rows_kernel", 1),
                                                ("s2_kernels.cu", "page_rows_kernel", 1)])
def test_paged_kernels_compile_without_spills(tmp_path, src, kernel, entries):
    """The kernels that read or write through a page table, the paged attn_kernel<128> instance among them, compile for
    sm_90a with no stack frame and no spill."""
    from internnav_b200 import build
    cmd = [_nvcc()] + build.FLAGS + ["-c", os.path.join(build.CSRC, src), "-o", str(tmp_path / "k.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found = re.findall(r"Function properties for (\S*%s\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads" % kernel, r.stderr)
    assert len(found) == entries, (len(found), r.stderr[-2000:])
    for name, stack, st, ld in found:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), "%s: %s bytes stack, %s / %s bytes spilled" % (name, stack, st, ld)
