"""Export of top-N lists (selfrec_b200/export.py) without a GPU: the manifest and name files, the reader and the
reassembly of the parts of a sharded export, the atomic publish (a stale temporary directory, a failing rank, a
replaced export), and the refusals.  The ranking itself is stubbed: each part's files are written from fixed arrays."""
import json
import os

import numpy as np
import pytest

from selfrec_b200 import checkpoint, export
from selfrec_b200._lib import SrbError

N = 4


def _model(tiny_conf, tiny_triples):
    from selfrec_b200.base.graph_recommender import GraphRecommender
    train, test = tiny_triples
    return GraphRecommender(tiny_conf("MF"), [list(t) for t in train], [list(t) for t in test])


def _lists(uids):
    """Deterministic fake lists of global user ids."""
    u = np.asarray(uids, dtype=np.int64)[:, None]
    return ((u * 7 + np.arange(N)) % 50).astype(np.int32), (-(u * 10 + np.arange(N))).astype(np.float32)


@pytest.fixture()
def fake_ranking(monkeypatch):
    def write_part(directory, g, uids, fn, n, score_dtype, chunk):
        ids, sc = _lists(uids)
        checkpoint.write_array(directory, f"users.{g}.npy", np.asarray(uids, dtype=np.int64))
        checkpoint.write_array(directory, f"ids.{g}.npy", ids)
        checkpoint.write_array(directory, f"scores.{g}.npy", sc)
    monkeypatch.setattr(export, "_write_part", write_part)


def _jobs(m, out, world):
    from selfrec_b200.shard_rank import owned_positions
    jobs = []
    for g in range(world):
        j = export._Job(m, out, top_n=N)
        pos, _ = owned_positions(j.uids, g, world)
        j.rank, j.world, j.uids = g, world, j.uids[pos]
        jobs.append(j)
    return jobs


@pytest.mark.parametrize("world", [1, 2, 3])
def test_manifest_reader_and_parts(tiny_conf, tiny_triples, fake_ranking, tmp_path, world):
    m = _model(tiny_conf, tiny_triples)
    path = export.run(_jobs(m, str(tmp_path), world), lambda ok: ok)
    assert path == os.path.join(str(tmp_path), f"MF-top{N}")
    man = json.load(open(os.path.join(path, "manifest.json")))
    d = m.data
    assert man == {"format": export.FORMAT_VERSION, "model": "MF", "U": d.user_num, "I": d.item_num, "d": None, "N": N,
                   "world": world, "pairs_fingerprint": checkpoint.pairs_fingerprint(d.pair_users, d.pair_items),
                   "score_dtype": "float32"}
    for g in range(world):
        u = np.load(os.path.join(path, f"users.{g}.npy"))
        assert np.all(np.diff(u) > 0) and np.all(u % world == g)
    names, ids, scores = export.read(path)
    want_ids, want_sc = _lists(np.arange(d.user_num))
    assert names == [d.id2user[u] for u in range(d.user_num)]
    assert np.array_equal(ids, want_ids) and np.array_equal(scores, want_sc)
    assert export.read_items(path) == [d.id2item[i] for i in range(d.item_num)]
    assert not [e for e in os.listdir(str(tmp_path)) if e.startswith(".")]


def test_stale_temporary_and_replaced_export(tiny_conf, tiny_triples, fake_ranking, tmp_path):
    m = _model(tiny_conf, tiny_triples)
    stale = tmp_path / f".MF-top{N}.tmp"
    stale.mkdir()
    (stale / "ids.0.npy").write_bytes(b"half a file")
    other = tmp_path / ".someone-else.tmp"  # not ours: left alone
    other.mkdir()
    path = export.run(_jobs(m, str(tmp_path), 1), lambda ok: ok)
    assert not stale.exists() and other.exists()
    (tmp_path / f"MF-top{N}" / "marker").write_text("old")
    export.run(_jobs(m, str(tmp_path), 2), lambda ok: ok)  # the same name again: replaced as a whole
    assert not os.path.exists(os.path.join(path, "marker"))
    assert json.load(open(os.path.join(path, "manifest.json")))["world"] == 2
    assert not os.path.exists(path + ".old")


def test_failure_publishes_nothing(tiny_conf, tiny_triples, fake_ranking, tmp_path, monkeypatch):
    m = _model(tiny_conf, tiny_triples)
    export.run(_jobs(m, str(tmp_path), 1), lambda ok: ok)
    before = export.read(os.path.join(str(tmp_path), f"MF-top{N}"))

    def broken(*a, **k):
        raise OSError("disk full")
    monkeypatch.setattr(export, "_write_part", broken)
    with pytest.raises(OSError):
        export.run(_jobs(m, str(tmp_path), 1), lambda ok: ok)
    assert not (tmp_path / f".MF-top{N}.tmp").exists()
    after = export.read(os.path.join(str(tmp_path), f"MF-top{N}"))
    assert before[0] == after[0] and np.array_equal(before[1], after[1])


def test_another_rank_failing_stops_this_one(tiny_conf, tiny_triples, fake_ranking, tmp_path):
    m = _model(tiny_conf, tiny_triples)
    calls = []

    def agree(ok):  # the all-reduce: this rank is fine, a peer failed in the write phase
        calls.append(ok)
        return len(calls) != 2
    with pytest.raises(SrbError, match="another rank failed"):
        export.run(_jobs(m, str(tmp_path), 1), agree)
    assert os.listdir(str(tmp_path)) == []


def test_refusals(tiny_conf, tiny_triples, tmp_path):
    m = _model(tiny_conf, tiny_triples)
    I = m.data.item_num
    for bad in (0, -1, I + 1):
        with pytest.raises(SrbError, match="topN"):
            export._Job(m, str(tmp_path), top_n=bad)
    with pytest.raises(SrbError, match="unknown user"):
        export._Job(m, str(tmp_path), users=[m.data.id2user[0], "no-such-user"])
    with pytest.raises(SrbError, match="chunk"):
        export._Job(m, str(tmp_path), chunk=0)
    j = export._Job(m, str(tmp_path), top_n=I, users=[m.data.id2user[3], m.data.id2user[1], m.data.id2user[3]])
    assert j.uids.tolist() == [1, 3] and j.n == I


def test_reader_refuses_other_formats(tmp_path):
    (tmp_path / "manifest.json").write_text(json.dumps({"format": 99}))
    with pytest.raises(SrbError, match="format"):
        export.read(str(tmp_path))
