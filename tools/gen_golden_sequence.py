"""Golden vectors of the sequential samplers and of batch_softmax_loss: runs the UNMODIFIED reference's
util/sampler.py (next_batch_sequence, next_batch_sequence_for_test) on its data/sequence.py Sequence, and its
util/loss_torch.py batch_softmax_loss under torch autograd on the CPU, and writes tests/golden/sequence.npz plus the
crafted sequential dataset it uses (seq_crafted_train.txt / seq_crafted_test.txt, `seq_id:item item ...` per line).
Needs a checkout of the reference and torch; run on a CPU machine:

    python tools/gen_golden_sequence.py --ref <reference checkout> [--out tests/golden]

Dataset: 40 items (a catalogue small enough that the negative draw of next_batch_sequence repeats), sequences shorter
than, equal to and longer than MAX_LEN, with repeated items, and length-1 sequences (Sequence drops them); names whose
string order differs from id order.  Samplers: two epochs of next_batch_sequence and one pass of
next_batch_sequence_for_test at MAX_LEN from random.seed(SEED), random.getstate() after each, and one test pass at the
default max_len.  Loss: batch_softmax_loss values and gradients at the CASES below, on the inputs that
tests/batch_softmax_oracle.case_inputs makes (they are not stored).
"""
import argparse
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from batch_softmax_oracle import case_inputs, grad_rows  # noqa: E402

SEED = 20261018
MAX_LEN = 8
BATCH = 8
# tag: (n, d, tau, salt, zero user rows, zero item rows)
CASES = {
    "a": (2048, 64, 0.07, 11, (), ()),
    "b": (2048, 128, 0.2, 13, (), ()),
    "c": (1, 64, 0.07, 17, (), ()),
    "d": (1, 128, 0.2, 19, (), ()),
    "e": (33, 128, 0.07, 23, (5, 20), (9, 20)),
    "f": (131, 64, 0.2, 29, (0,), ()),
}


def crafted_lines():
    rng = np.random.default_rng(SEED)
    items = [f"it{(37 * k) % 101}" for k in range(1, 41)]
    lengths = [2, 3, 7, 8, 9, 12, 20, 5, 2, 15, 8, 6, 1, 4, 30, 9, 10, 3, 1, 11, 7, 16, 2, 8, 25, 6, 13, 4, 9, 2, 1, 18]
    train, test = [], []
    for k, ln in enumerate(lengths):
        name = f"s{(k * 7) % 50}x"
        seq = [items[j] for j in rng.integers(0, 12 + k, size=ln) % len(items)]
        if ln >= 4:
            seq[2] = seq[0]  # a repeated item
        train.append(f"{name}:{' '.join(seq)}\n")
        test.append(f"{name}:{items[int(rng.integers(len(items)))]}\n")
    test.append("ghost:it5\n")  # a sequence unknown to training
    return train, test


def epoch_arrays(batches):
    cols = list(zip(*batches))
    return [np.concatenate(c) for c in cols], np.array([len(b[-1]) for b in batches])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", required=True, help="root of a Coder-Yu/SELFRec checkout")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden"))
    args = ap.parse_args()
    out = os.path.abspath(args.out)
    train_lines, test_lines = crafted_lines()
    for name, lines in (("seq_crafted_train.txt", train_lines), ("seq_crafted_test.txt", test_lines)):
        with open(os.path.join(out, name), "w") as f:
            f.writelines(lines)
    sys.path.insert(0, os.path.abspath(args.ref))
    import torch
    from data.loader import FileIO
    from data.sequence import Sequence
    from util.loss_torch import batch_softmax_loss
    from util.sampler import next_batch_sequence, next_batch_sequence_for_test

    fx = dict(meta=np.array(str(dict(python=sys.version.split()[0], numpy=np.__version__, torch=torch.__version__))),
              seed=np.array(SEED), max_len=np.array(MAX_LEN), batch=np.array(BATCH))
    train = FileIO.load_data_set(os.path.join(out, "seq_crafted_train.txt"), "sequential")
    test = FileIO.load_data_set(os.path.join(out, "seq_crafted_test.txt"), "sequential")
    data = Sequence({}, train, test)
    fx["item_num"] = np.array(data.item_num)
    fx["seq_names"] = np.array([s for s, _ in data.original_seq])
    fx["seq_ptr"] = np.cumsum([0] + [len(x) for _, x in data.original_seq])
    fx["seq_items"] = np.concatenate([x for _, x in data.original_seq])
    random.seed(SEED)
    for e in range(2):
        (seq, pos, y, neg, seq_len), sizes = epoch_arrays(list(next_batch_sequence(data, BATCH, max_len=MAX_LEN)))
        fx.update({f"e{e}_seq": seq, f"e{e}_pos": pos, f"e{e}_y": y, f"e{e}_neg": neg, f"e{e}_seq_len": seq_len,
                   f"e{e}_sizes": sizes, f"e{e}_state": np.array(random.getstate()[1], dtype=np.uint32)})
    (seq, pos, seq_len), sizes = epoch_arrays(list(next_batch_sequence_for_test(data, BATCH, max_len=MAX_LEN)))
    fx.update(t_seq=seq, t_pos=pos, t_seq_len=seq_len, t_sizes=sizes, t_state=np.array(random.getstate()[1], dtype=np.uint32))
    (seq, pos, seq_len), sizes = epoch_arrays(list(next_batch_sequence_for_test(data, 5)))
    fx.update(t50_seq=seq, t50_pos=pos, t50_seq_len=seq_len, t50_sizes=sizes)

    torch.set_num_threads(1)
    for tag, (n, d, tau, salt, zu, zi) in CASES.items():
        u, i = case_inputs(n, d, salt, zu, zi)
        tu, ti = torch.from_numpy(u).requires_grad_(True), torch.from_numpy(i).requires_grad_(True)
        loss = batch_softmax_loss(tu, ti, tau)
        gu, gi = torch.autograd.grad(loss, (tu, ti))
        rows = grad_rows(n)
        fx.update({f"bsm_{tag}_n": np.array(n), f"bsm_{tag}_d": np.array(d), f"bsm_{tag}_tau": np.array(tau),
                   f"bsm_{tag}_salt": np.array(salt), f"bsm_{tag}_zero_users": np.array(zu, dtype=np.int64),
                   f"bsm_{tag}_zero_items": np.array(zi, dtype=np.int64),
                   f"bsm_{tag}_sum": np.array([u.astype(np.float64).sum(), i.astype(np.float64).sum()]),
                   f"bsm_{tag}_loss": np.array(loss.item()), f"bsm_{tag}_rows": rows,
                   f"bsm_{tag}_gu": gu.numpy()[rows], f"bsm_{tag}_gi": gi.numpy()[rows]})
        print(tag, "loss", loss.item())
    np.savez_compressed(os.path.join(out, "sequence.npz"), **fx)
    print("wrote", os.path.join(out, "sequence.npz"))


if __name__ == "__main__":
    main()
