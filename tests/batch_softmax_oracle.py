"""Float64 restatement of batch_softmax_loss (reference util/loss_torch.py:25-32) and its autograd gradient, plus the
inputs of the tests/golden/sequence.npz loss cases.  Test infrastructure, like oracle/oracle.py's infonce()."""
import numpy as np

EPS = 1e-5  # the reference's 10e-6


def batch_softmax_loss(user_emb, item_emb, temperature):
    """Returns (loss, d loss / d user_emb, d loss / d item_emb) in float64.  The softmax is taken in log-sum-exp form;
    where the reference's unshifted exp(S) stays finite (temperature >= 1/88) the two agree."""
    u, i = np.asarray(user_emb, dtype=np.float64), np.asarray(item_emb, dtype=np.float64)
    nu = np.maximum(np.sqrt((u ** 2).sum(1, keepdims=True)), 1e-12)
    ni = np.maximum(np.sqrt((i ** 2).sum(1, keepdims=True)), 1e-12)
    a, b = u / nu, i / ni
    S = a @ b.T / temperature
    m = S.max(1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(S - m).sum(1))
    n = S.shape[0]
    p = np.exp(np.diag(S) - lse)
    loss = np.mean(-np.log(p + EPS))
    c = p / (p + EPS)
    G = c[:, None] * (np.exp(S - lse[:, None]) - np.eye(n)) / n / temperature  # d loss / d (a b^T)
    da, db = G @ b, G.T @ a
    da = (da - a * (a * da).sum(1, keepdims=True)) / nu
    db = (db - b * (b * db).sum(1, keepdims=True)) / ni
    return loss, da, db


def _unit_floats(n, d, salt):
    """[n, d] float32 in [-1, 1), multiples of 2^-23: splitmix64 of (salt, element index).  Integer arithmetic only, so
    every numpy on every platform makes the same bits, and the fixture need not store its inputs."""
    with np.errstate(over="ignore"):
        z = np.arange(n * d, dtype=np.uint64) + np.uint64(salt) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    v = (z >> np.uint64(40)).astype(np.int64) - (1 << 23)
    return (v.astype(np.float32) / np.float32(1 << 23)).reshape(n, d)


def case_inputs(n, d, salt, zero_users=(), zero_items=()):
    """The (user_emb, item_emb) of one loss case: item rows lean towards their user rows, so the diagonal of S stands
    out as it does for trained towers; the listed rows are zero."""
    u = _unit_floats(n, d, salt)
    i = (u + np.float32(0.5) * _unit_floats(n, d, salt + 1)).astype(np.float32)
    u[list(zero_users)] = 0
    i[list(zero_items)] = 0
    return u, i


def grad_rows(n):
    """The rows whose gradients the fixture keeps: all of them up to 256, else the first and last tiles' edges and a
    stride through the middle."""
    if n <= 256:
        return np.arange(n)
    edges = [r for e in (0, 64, 128, n - 64, n) for r in range(e - 4, e + 4)]
    return np.unique(np.clip(np.r_[edges, np.arange(0, n, 97)], 0, n - 1))
