"""Ranking metrics with the output format of util/evaluation.py:135-162.

ranking_evaluation(origin, res, N) keeps the reference's string protocol (fast_evaluation
re-parses it, graph_recommender.py:84-86): for each n a 'Top n' line followed by
'Hit Ratio:', 'Precision:', 'Recall:', 'NDCG:' lines, values rounded to 5 decimals.
"""
import math


def _hits(origin, predicted):
    return {u: len(set(origin[u]).intersection(it[0] for it in predicted[u])) for u in origin}


def ranking_evaluation(origin, res, N):
    measure = []
    for n in N:
        predicted = {u: res[u][:n] for u in res}
        if len(origin) != len(predicted):
            print("The Lengths of test set and predicted set do not match!")
            exit(-1)
        hits = _hits(origin, predicted)
        total = sum(len(origin[u]) for u in origin)
        hit_sum = sum(hits.values())
        hr = round(hit_sum / total, 5)
        prec = round(hit_sum / (len(hits) * n), 5)
        rec_list = [hits[u] / len(origin[u]) for u in hits]
        recall = round(sum(rec_list) / len(rec_list), 5)
        ndcg_sum = 0
        for u in predicted:
            dcg = sum(1.0 / math.log(r + 2, 2) for r, it in enumerate(predicted[u]) if it[0] in origin[u])
            idcg = sum(1.0 / math.log(r + 2, 2) for r in range(min(len(origin[u]), n)))
            ndcg_sum += dcg / idcg
        ndcg = round(ndcg_sum / len(predicted), 5)
        measure.append("Top " + str(n) + "\n")
        measure += ["Hit Ratio:" + str(hr) + "\n", "Precision:" + str(prec) + "\n", "Recall:" + str(recall) + "\n",
                    "NDCG:" + str(ndcg) + "\n"]
    return measure


def ranking_evaluation_from_masks(n_test, masks, N):
    """Same strings as ranking_evaluation, from per-user hit masks (bit r of masks[q] = the item at rank r is
    a test item of that user; ops.rank_hit_masks) and n_test[q] = len(origin[user]), both in test-set order.
    masks is one 64-bit word per user, or [n, W] words per user for lists longer than 64 (bit r % 64 of word
    r // 64).
    Every float expression is the reference's (util/evaluation.py:9-15, 45-53, 85-97, 135-162) evaluated on
    the same operands in the same order, so the rounded values are identical."""
    n_test = [int(x) for x in n_test]
    if getattr(masks, "ndim", 1) == 2:
        masks = [sum((int(w) & 0xFFFFFFFFFFFFFFFF) << (64 * j) for j, w in enumerate(row)) for row in masks]
    else:
        masks = [int(m) & 0xFFFFFFFFFFFFFFFF for m in masks]
    if len(n_test) != len(masks):
        print("The Lengths of test set and predicted set do not match!")
        exit(-1)
    measure = []
    total = sum(n_test)
    for n in N:
        cut = (1 << n) - 1
        hits = [bin(m & cut).count("1") for m in masks]
        hit_sum = sum(hits)
        hr = round(hit_sum / total, 5)
        prec = round(hit_sum / (len(hits) * n), 5)
        rec_list = [h / t for h, t in zip(hits, n_test)]
        recall = round(sum(rec_list) / len(rec_list), 5)
        idcg_cache = {}
        ndcg_sum = 0
        for m, t in zip(masks, n_test):
            m &= cut
            dcg = sum(1.0 / math.log(r + 2, 2) for r in range(n) if (m >> r) & 1) if m else 0
            k = min(t, n)
            if k not in idcg_cache:
                idcg_cache[k] = sum(1.0 / math.log(r + 2, 2) for r in range(k))
            ndcg_sum += dcg / idcg_cache[k]
        ndcg = round(ndcg_sum / len(masks), 5)
        measure.append("Top " + str(n) + "\n")
        measure += ["Hit Ratio:" + str(hr) + "\n", "Precision:" + str(prec) + "\n", "Recall:" + str(recall) + "\n",
                    "NDCG:" + str(ndcg) + "\n"]
    return measure
