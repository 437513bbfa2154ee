"""Long top-k lists (33..256) without a GPU: the multi-word hit-mask metrics against ranking_evaluation, the
workspace arithmetic and dispatch rule of the tensor-core route, and a numpy model of its running-threshold candidate
buffers (csrc/score_topk_tc.cu, tc_score_kernel<D, true>) showing that a certified user's candidates hold the true
top k and every item tied with the k-th."""
import numpy as np
import pytest


def _lists(rng, n_users, n_items, k):
    test = {f"u{u}": {f"i{i}": 1 for i in rng.choice(n_items, int(rng.integers(1, 40)), replace=False)} for u in range(n_users)}
    rec = {u: [(f"i{i}", float(-r)) for r, i in enumerate(rng.choice(n_items, k, replace=False))] for u in test}
    for u in list(test)[::7]:  # some users with their test items ranked first (lists stay duplicate-free)
        t = list(test[u])
        rest = [f"i{i}" for i in rng.permutation(n_items) if f"i{i}" not in test[u]]
        rec[u] = [(it, float(-r)) for r, it in enumerate((t + rest)[:k])]
    return test, rec


@pytest.mark.parametrize("k", [1, 63, 64, 65, 127, 128, 129, 200, 255, 256])
def test_multiword_masks_equal_ranking_evaluation(k):
    from selfrec_b200.util.evaluation import ranking_evaluation, ranking_evaluation_from_masks
    rng = np.random.default_rng(k)
    test, rec = _lists(rng, 120, 400, k)
    words = (k + 63) // 64
    masks = np.zeros((len(test), words), np.uint64)
    for q, u in enumerate(test):
        for r, (it, _) in enumerate(rec[u]):
            if it in test[u]:
                masks[q, r // 64] |= np.uint64(1 << (r % 64))
    n_test = [len(test[u]) for u in test]
    for cut in sorted({1, min(k, 20), k}):
        want = ranking_evaluation(test, rec, [cut])
        assert ranking_evaluation_from_masks(n_test, masks, [cut]) == want
        if words == 1:  # the one-word form is unchanged
            assert ranking_evaluation_from_masks(n_test, masks[:, 0], [cut]) == want


def _cap(k):
    return (2 * k + 256 + 31) // 32 * 32


def _align(x):
    return (x + 255) // 256 * 256


def test_workspace_arithmetic(built_lib):
    """Lists of 33..256 add two [n_q][2][cap(k)] buffers (score, id) after the fallback counter; no term grows with
    n_q * n_items, the counter offset does not move, and lists of k <= 32 keep the same workspace."""
    lib = built_lib
    for n_q, n_items in ((1, 1024), (1000, 5000), (31668, 38048)):
        base = lib.srb_topk_workspace_bytes(n_q, n_items, 64, 20)
        assert lib.srb_topk_workspace_bytes(n_q, n_items, 64, 1) == base == lib.srb_topk_workspace_bytes(n_q, n_items, 64, 32)
        for k in (33, 50, 100, 256):
            assert lib.srb_topk_workspace_bytes(n_q, n_items, 64, k) - base == 2 * _align(n_q * 2 * _cap(k) * 4)
            assert lib.srb_topk_workspace_bytes(n_q, n_items, 128, k) - lib.srb_topk_workspace_bytes(n_q, n_items, 64, k) == \
                ((n_q + 255) // 256 * 256 + 256) * 64 * 4
        assert 0 <= lib.srb_topk_fallback_count_offset(n_q, n_items) < base
    # the long-list part does not depend on the catalogue
    for k in (33, 256):
        grow = [lib.srb_topk_workspace_bytes(5000, n, 128, k) - lib.srb_topk_workspace_bytes(5000, n, 128, 20) for n in (1024, 10 ** 6)]
        assert grow[0] == grow[1]


def test_dispatch_rule():
    from selfrec_b200 import ops
    lr = ops.long_list_route
    assert lr(64, 1024, 33) and lr(128, 38048, 256) and lr(64, 10 ** 6, 100)
    assert not lr(64, 1024, 32)           # short lists: the existing 2 x 24 candidate lists
    assert not lr(64, 1024, 257)          # above 256: dense rows
    assert not lr(64, 1023, 100)          # small catalogue: dense rows unless impl 2 is asked for
    assert lr(64, 1023, 100, impl=2) and not lr(64, 4096, 100, impl=1)
    for d in (16, 32, 256):
        assert not lr(d, 38048, 100)


def _find_k_largest(scores, ids, k):
    """find_k_largest's heap over (score, id) in the given (id) order: seeded with the first k, then a strictly
    greater score replaces the heap's smallest (score, id)."""
    import heapq
    heap = [(float(s), int(i)) for s, i in zip(scores[:k], ids[:k])]
    heapq.heapify(heap)
    for s, i in zip(scores[k:], ids[k:]):
        if float(s) > heap[0][0]:
            heapq.heapreplace(heap, (float(s), int(i)))
    return {i for _, i in heap}


def _okey(s):
    s = np.where(s == 0, np.float32(0), s).astype(np.float32)
    b = s.view(np.uint32)
    return np.where(b & 0x80000000, ~b, b | 0x80000000).astype(np.uint32)


def _ofloat(v):
    v = np.uint32(v)
    return np.array([(v & 0x7FFFFFFF) if (v & 0x80000000) else ~v], np.uint32).view(np.float32)[0]


def _half_buffer(approx, ids, k, cap, two_e):
    """The kernel's per-half loop: append approx > thr, compact a full buffer (thr := max(thr, lb_k - 2E), lb_k the
    20-bit lower bound of the k-th best key), overflow when a compaction frees less than a quarter."""
    thr, bs, bi = np.float32(-np.inf), [], []
    for s, i in zip(approx, ids):
        if not s > thr:
            continue
        bs.append(s)
        bi.append(i)
        if len(bs) == cap:
            keys = _okey(np.array(bs, np.float32))
            v = 0
            for b in range(31, 11, -1):
                t = v | (1 << b)
                if int((keys >= t).sum()) >= k:
                    v = t
            if v:
                thr = max(thr, np.float32(_ofloat(v) - two_e))
            keep = [j for j in range(cap) if bs[j] > thr]
            bs, bi = [bs[j] for j in keep], [bi[j] for j in keep]
            if len(bs) > cap - cap // 4:
                return None, np.float32(np.inf)
    return (np.array(bs, np.float32), np.array(bi, np.int64)), thr


@pytest.mark.parametrize("k", [33, 100, 256])
@pytest.mark.parametrize("kind", ["gauss", "ties", "common"])
def test_running_threshold_certificate(k, kind):
    """Approximate scores within E of the exact ones: whenever the certificate max(thr) + E < exact k-th passes, the
    candidates contain every item scoring at or above the exact k-th (the true top k and every item tied with the
    k-th), so find_k_largest over the candidates in id order keeps what it keeps over the whole catalogue."""
    rng = np.random.default_rng(k + len(kind))
    n_items, cap = 6000, _cap(k)
    certified = 0
    for trial in range(6):
        if kind == "gauss":
            exact = rng.standard_normal(n_items).astype(np.float32)
        elif kind == "ties":
            exact = rng.integers(-40, 40, n_items).astype(np.float32) / 8
        else:
            exact = (1.0 + 1e-5 * rng.standard_normal(n_items)).astype(np.float32)
        E = np.float32(2.0 ** -9 * np.abs(exact).max())
        approx = (exact + rng.uniform(-1, 1, n_items).astype(np.float32) * E * np.float32(0.999)).astype(np.float32)
        top = _find_k_largest(exact, np.arange(n_items), k)
        kth = np.sort(exact)[::-1][k - 1]
        ties = set(np.flatnonzero(exact == kth).tolist())
        cand, thr = set(), np.float32(-np.inf)
        ok = True
        for h in range(2):  # two column halves: 64-item groups alternate between them
            sel = np.flatnonzero(((np.arange(n_items) // 64) % 2) == h)
            buf, t = _half_buffer(approx[sel], sel, k, cap, np.float32(2 * E))
            if buf is None:
                ok = False
                break
            cand |= set(buf[1].tolist())
            thr = max(thr, t)
            # invariant: every item of the half above the final threshold is a candidate
            assert set(sel[approx[sel] > t].tolist()) <= set(buf[1].tolist())
        if not ok or len(cand) < k:
            continue
        c = np.array(sorted(cand))
        if np.float32(thr + E) < np.sort(exact[c])[::-1][k - 1]:
            certified += 1
            assert top <= cand and ties <= cand
            assert _find_k_largest(exact[c], c, k) == top
    if kind == "gauss":
        assert certified == 6
