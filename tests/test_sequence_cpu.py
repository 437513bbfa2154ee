"""The sequential samplers and batch_softmax_loss of the drop-in modules, on the CPU: the util/sampler.py mirror and the
float64 restatement of batch_softmax_loss against tests/golden/sequence.npz (made by tools/gen_golden_sequence.py from
the reference), and the names the reference's model and base files import once install() has aliased the modules."""
import importlib
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import pytest

import batch_softmax_oracle as bso

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _sequence_data(fx):
    """data/sequence.py's Sequence on the crafted file, restated: sequences of two items or more, in file order, item
    ids from 1 in order of first appearance.  Checked against the reference's original_seq."""
    from selfrec_b200.data.loader import FileIO
    train = FileIO.load_data_set(os.path.join(GOLDEN, "seq_crafted_train.txt"), "sequential")
    ids, original = {}, []
    for name, items in train.items():
        if len(items) < 2:
            continue
        for it in items:
            ids.setdefault(it, len(ids) + 1)
        original.append((name, [ids[it] for it in items]))
    assert [s for s, _ in original] == list(fx["seq_names"])
    assert np.array_equal(np.concatenate([x for _, x in original]), fx["seq_items"])
    assert np.array_equal(np.cumsum([0] + [len(x) for _, x in original]), fx["seq_ptr"])
    assert len(ids) == int(fx["item_num"])
    return SimpleNamespace(original_seq=original, item_num=len(ids))


def _collect(batches):
    cols = list(zip(*batches))
    return [np.concatenate(c) for c in cols], [len(b[-1]) for b in batches]


def _state():
    return np.array(random.getstate()[1], dtype=np.uint32)


def test_sequence_samplers_match_reference(golden):
    from selfrec_b200.util.sampler import next_batch_sequence, next_batch_sequence_for_test
    fx = golden("sequence.npz")
    data = _sequence_data(fx)
    max_len, batch = int(fx["max_len"]), int(fx["batch"])
    random.seed(int(fx["seed"]))
    for e in range(2):
        batches = list(next_batch_sequence(data, batch, max_len=max_len))
        for b in batches:
            assert len(b) == 5 and all(a.dtype == np.int64 for a in b)
            assert b[0].shape == (len(b[4]), max_len)
        (seq, pos, y, neg, seq_len), sizes = _collect(batches)
        for got, key in ((seq, "seq"), (pos, "pos"), (y, "y"), (neg, "neg"), (seq_len, "seq_len")):
            assert np.array_equal(got, fx[f"e{e}_{key}"]), (e, key)
        assert sizes == list(fx[f"e{e}_sizes"])
        assert np.array_equal(_state(), fx[f"e{e}_state"]), e  # the negative draws consumed the same stream
    # the sequence order the shuffles left is not the file's: the epochs really are shuffled
    assert not np.array_equal(fx["e0_seq"], fx["t_seq"])
    (seq, pos, seq_len), sizes = _collect(list(next_batch_sequence_for_test(data, batch, max_len=max_len)))
    assert np.array_equal(seq, fx["t_seq"]) and np.array_equal(pos, fx["t_pos"]) and np.array_equal(seq_len, fx["t_seq_len"])
    assert sizes == list(fx["t_sizes"])
    assert np.array_equal(_state(), fx["t_state"])  # the test batches draw nothing
    (seq, pos, seq_len), sizes = _collect(list(next_batch_sequence_for_test(data, 5)))  # default max_len = 50
    assert seq.shape[1] == 50 and sizes == list(fx["t50_sizes"])
    assert np.array_equal(seq, fx["t50_seq"]) and np.array_equal(pos, fx["t50_pos"]) and np.array_equal(seq_len, fx["t50_seq_len"])


def fp32_floor(u, i, tau):
    """The gradient error of any fp32 evaluation near a zero loss gradient, as in test_infonce_batch_sizes: G_rr =
    c_r (P_rr - 1) carries an absolute error ~ eps32 / tau, through 1/(n tau), a unit-vector entry (1/sqrt(d)) and
    1/||v|| (the smallest non-zero row)."""
    n, d = u.shape
    norms = np.linalg.norm(np.concatenate([u, i]).astype(np.float64), axis=1)
    return 3 * 1.2e-7 / tau / (n * tau) / np.sqrt(d) / norms[norms > 0].min()


def _cases(fx):
    return sorted({k.split("_")[1] for k in fx.files if k.startswith("bsm_")})


def test_batch_softmax_oracle_matches_reference_autograd(golden):
    fx = golden("sequence.npz")
    tags = _cases(fx)
    assert len(tags) >= 6
    for tag in tags:
        g = lambda k: fx[f"bsm_{tag}_{k}"]
        u, i = bso.case_inputs(int(g("n")), int(g("d")), int(g("salt")), g("zero_users"), g("zero_items"))
        assert np.array_equal(g("sum"), [u.astype(np.float64).sum(), i.astype(np.float64).sum()]), tag
        loss, gu, gi = bso.batch_softmax_loss(u, i, float(g("tau")))
        ref = float(g("loss"))
        assert abs(loss - ref) <= 2e-5 * max(abs(ref), 1e-3), (tag, loss, ref)
        rows = g("rows")
        cond = fp32_floor(u, i, float(g("tau")))
        for mine, key in ((gu[rows], "gu"), (gi[rows], "gi")):
            want = g(key)
            # per-row scale: a zero row's gradient is 1/eps = 1e12 times its neighbours'
            atol = 2e-6 * np.abs(want).max(1, keepdims=True) + cond
            assert (np.abs(mine - want) <= 2e-5 * np.abs(want) + atol).all(), (tag, key)


def test_batch_softmax_oracle_is_finite_where_the_reference_overflows():
    """Below temperature 1/88.7 the reference's exp(S / tau) overflows fp32; the log-sum-exp form is the limit of the
    exact loss, which the float64 reference form still reaches at this tau."""
    u, i = bso.case_inputs(64, 32, 5)
    tau = 1 / 120
    loss, gu, gi = bso.batch_softmax_loss(u, i, tau)
    assert np.isfinite(loss) and np.isfinite(gu).all() and np.isfinite(gi).all()
    a = u / np.linalg.norm(u.astype(np.float64), axis=1, keepdims=True)
    b = i / np.linalg.norm(i.astype(np.float64), axis=1, keepdims=True)
    e = np.exp(a @ b.T / tau)  # float64: e^120 is representable
    assert abs(loss - np.mean(-np.log(np.diag(e) / e.sum(1) + 1e-5))) <= 1e-9 * abs(loss)
    with np.errstate(over="ignore", invalid="ignore"):
        e32 = np.exp((a @ b.T / tau).astype(np.float32))
        assert not np.isfinite(np.diag(e32) / e32.sum(1)).all()  # what an fp32 unshifted sum gives


# Every name the reference's model/*/*.py and base/*.py import from a module install() aliases (module -> names).
# Written out here because the tests do not read the reference tree.
REFERENCE_IMPORTS = {
    "base.graph_recommender": ["GraphRecommender"],  # model/graph/*.py
    "base.torch_interface": ["TorchGraphInterface"],  # BUIR, LightGCN, MixGCF, NCL, SGL, SimGCL, XSimGCL
    "data.ui_graph": ["Interaction"],  # base/graph_recommender.py:2
    "data.loader": ["FileIO"],  # base/graph_recommender.py:5, SELFRec.py:1
    "util.evaluation": ["ranking_evaluation"],  # base/graph_recommender.py:7, base/seq_recommender.py:4
    "util.sampler": [
        "next_batch_pairwise",  # model/graph/*.py
        "next_batch_sequence",  # SASRec.py:5, BERT4Rec.py:6, CL4SRec.py:5
        "next_batch_sequence_for_test",  # base/seq_recommender.py:5
    ],
    "util.loss_torch": [
        "bpr_loss", "l2_reg_loss",  # DirectAU, LightGCN, MF, MixGCF, NCL, SGL, SimGCL, XSimGCL; l2 also the sequential models
        "InfoNCE",  # NCL, SGL, SimGCL, XSimGCL, SSL4Rec.py:6, CL4SRec.py:7
        "batch_softmax_loss",  # SSL4Rec.py:6, CL4SRec.py:7
    ],
}


@pytest.mark.parametrize("fused_models", [True, False])
def test_install_resolves_every_reference_import(built_lib, fused_models):
    import selfrec_b200
    names = selfrec_b200.install(fused_models=fused_models)
    try:
        assert set(REFERENCE_IMPORTS) <= set(names)
        for alias, wanted in REFERENCE_IMPORTS.items():
            mod = importlib.import_module(alias)
            assert mod is sys.modules[alias] and mod.__name__.startswith("selfrec_b200.")
            for name in wanted:
                assert callable(getattr(mod, name, None)), f"from {alias} import {name}"
    finally:
        for n in names:
            sys.modules.pop(n, None)
