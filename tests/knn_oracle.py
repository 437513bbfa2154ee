"""Float64 restatement of the neighbourhood baselines (reference model/graph/ItemKNN.py, model/graph/UserKNN.py) and of
find_k_largest (util/algorithm.py:144-156) on float64 rows, written from the rules in DESIGN §11.  Test infrastructure:
numpy elementwise operations are single correctly rounded IEEE double operations, so every value here has the
reference's bits, and the GPU tests compare with `==`."""
import heapq

import numpy as np
import scipy.sparse as sp


def neighbours(ptr, idx, n_cols, rank, topk, shrinkage):
    """Rows of the binary CSR (ptr, idx) against each other: ids int32 [n, topk] (-1 past counts), sims float64 [n, topk]
    (0 past counts), counts int32 [n].  Key: sim descending, then rank of the other row descending."""
    n = len(ptr) - 1
    A = sp.csr_matrix((np.ones(len(idx), dtype=np.int64), idx, ptr), shape=(n, n_cols))
    C = (A @ A.T).tocsr()
    deg = np.diff(ptr).astype(np.int64)
    ids = np.full((n, topk), -1, dtype=np.int32)
    sims = np.zeros((n, topk), dtype=np.float64)
    counts = np.zeros(n, dtype=np.int32)
    for a in range(n):
        b = C.indices[C.indptr[a]:C.indptr[a + 1]]
        c = C.data[C.indptr[a]:C.indptr[a + 1]]
        keep = (b != a) & (c > 0)
        b, c = b[keep], c[keep]
        raw = c / (np.sqrt(np.float64(deg[a])) * np.sqrt(deg[b].astype(np.float64)) + 1e-8)
        sim = (c / (c + shrinkage)) * raw
        order = np.lexsort((-rank[b].astype(np.int64), -sim))[:topk]
        counts[a] = len(order)
        ids[a, :len(order)] = b[order]
        sims[a, :len(order)] = sim[order]
    return ids, sims, counts


def score_row(mode, u, n_items, table, seq_ptr, seq_idx):
    """predict(u) as a float64 [n_items] row.  mode "item": the sims of the neighbours of each of u's items, items in
    seq (training_set_u) order; mode "user": each neighbour's sim added to all its items, neighbours in list order.
    Then acc / (acc + 1e-8)."""
    ids, sims, counts = table
    acc = np.zeros(n_items, dtype=np.float64)
    if mode == "item":
        for i in seq_idx[seq_ptr[u]:seq_ptr[u + 1]]:
            n = counts[i]
            acc[ids[i, :n]] += sims[i, :n]  # distinct destinations within one list
    else:
        for t in range(counts[u]):
            v = ids[u, t]
            acc[seq_idx[seq_ptr[v]:seq_ptr[v + 1]]] += sims[u, t]
    return acc / (acc + 1e-8)


def _argsort_desc(A):
    """numba's list.sort(key=score, reverse=True): its quicksort argsort with LT(a, b) = a > b."""
    n = len(A)
    R = list(range(n))
    if n < 2:
        return R

    def insertion(low, high):
        for i in range(low + 1, high + 1):
            k = R[i]
            v = A[k]
            j = i
            while j > low and v > A[R[j - 1]]:
                R[j] = R[j - 1]
                j -= 1
            R[j] = k

    def partition(low, high):
        mid = (low + high) >> 1
        if A[R[mid]] > A[R[low]]:
            R[low], R[mid] = R[mid], R[low]
        if A[R[high]] > A[R[mid]]:
            R[high], R[mid] = R[mid], R[high]
        if A[R[mid]] > A[R[low]]:
            R[low], R[mid] = R[mid], R[low]
        pivot = A[R[mid]]
        R[high], R[mid] = R[mid], R[high]
        i, j = low, high - 1
        while True:
            while i < high and A[R[i]] > pivot:
                i += 1
            while j >= low and pivot > A[R[j]]:
                j -= 1
            if i >= j:
                break
            R[i], R[j] = R[j], R[i]
            i += 1
            j -= 1
        R[i], R[high] = R[high], R[i]
        return i

    stack = [(0, n - 1)]
    while stack:
        low, high = stack.pop()
        while high - low >= 15:
            i = partition(low, high)
            if high - i > i - low:
                if high > i:
                    stack.append((i + 1, high))
                high = i - 1
            else:
                if i > low:
                    stack.append((low, i - 1))
                low = i + 1
        insertion(low, high)
    return R


def find_k_largest(K, row):
    """(ids, scores) of util/algorithm.py:144-156 on a float64 row: heapq over (score, id) tuples, then the argsort."""
    row = [float(x) for x in row]
    heap = [(s, i) for i, s in enumerate(row[:K])]
    heapq.heapify(heap)
    for i in range(K, len(row)):
        if row[i] > heap[0][0]:
            heapq.heapreplace(heap, (row[i], i))
    order = _argsort_desc([h[0] for h in heap])
    return np.array([heap[r][1] for r in order], dtype=np.int32), np.array([heap[r][0] for r in order], dtype=np.float64)


def rank_users(mode, uids, n_items, table, seq_ptr, seq_idx, rated_ptr, rated_idx, K):
    """find_k_largest(K, masked predict row) per user id: (ids int32 [n, K], scores float64 [n, K])."""
    ids = np.empty((len(uids), K), dtype=np.int32)
    sc = np.empty((len(uids), K), dtype=np.float64)
    for q, u in enumerate(uids):
        row = score_row(mode, u, n_items, table, seq_ptr, seq_idx)
        row[rated_idx[rated_ptr[u]:rated_ptr[u + 1]]] = -10e8
        ids[q], sc[q] = find_k_largest(K, row)
    return ids, sc


def model_inputs(pair_users, pair_items, n_users, n_items, user_names, item_names):
    """What both models read, from the training pairs in file order: the training_set_u lists, the item -> user CSR and
    the name ranks.  Restated here independently of selfrec_b200.knn."""
    seen, rows = set(), [[] for _ in range(n_users)]
    for u, i in zip(np.asarray(pair_users).tolist(), np.asarray(pair_items).tolist()):
        if (u, i) not in seen:
            seen.add((u, i))
            rows[u].append(i)
    cols = [[] for _ in range(n_items)]
    for u, r in enumerate(rows):
        for i in r:
            cols[i].append(u)
    csr = lambda lists: (np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32),
                         np.array([v for x in lists for v in x], dtype=np.int32))
    rk = lambda names: np.argsort(np.array(sorted(range(len(names)), key=names.__getitem__))).astype(np.int32)
    seq_ptr, seq_idx = csr(rows)
    iu_ptr, iu_idx = csr([sorted(c) for c in cols])
    return dict(seq_ptr=seq_ptr, seq_idx=seq_idx, iu_ptr=iu_ptr, iu_idx=iu_idx, user_rank=rk(user_names), item_rank=rk(item_names))


def model_table(kind, inp, n_users, n_items, topk, shrinkage):
    """The neighbour table of ItemKNN (kind "item") or UserKNN ("user")."""
    if kind == "item":
        return neighbours(inp["iu_ptr"], inp["iu_idx"], n_users, inp["item_rank"], topk, shrinkage)
    return neighbours(inp["seq_ptr"], inp["seq_idx"], n_items, inp["user_rank"], topk, shrinkage)
