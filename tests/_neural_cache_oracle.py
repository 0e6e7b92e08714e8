"""Float64 numpy restatement of the neural-cache evaluation (Grave, Joulin & Usunier 2017; DESIGN.md section 12).

`NeuralCache(size, batch)` keeps, per stream, the last `size` pairs (key, token) across calls, exactly as the ring of
zrb_cache does: key = half_rn(h) of the last layer's output, token = the target at that position.  `step(h, y, theta,
lam, row_loss)` appends a [T,B] window and returns p_cache, the mixed row losses and the window loss.  The model-level
tests feed it `oracle.lstm_lm_oracle.model_fwd`'s cache["fc_in"] and the row losses of its scores.
"""
import numpy as np


def half_round(a):
    """half_rn(a) as float64 (numpy's float16 conversion rounds to nearest even)."""
    return np.asarray(a, dtype=np.float64).astype(np.float16).astype(np.float64)


def mix_row_loss(r, p_cache, empty, lam):
    """-log((1 - lam) exp(-r) + lam p_cache) in log-add-exp form; a row with an empty cache keeps r."""
    r = np.asarray(r, dtype=np.float64)
    if lam == 0.0:
        return r.copy()
    with np.errstate(divide="ignore"):
        mixed = -np.logaddexp(np.log1p(-lam) - r, np.log(lam) + np.log(p_cache))
    return np.where(empty, r, mixed)


class NeuralCache:
    def __init__(self, size, batch):
        assert size >= 1 and batch >= 1
        self.W, self.B = int(size), int(batch)
        self.reset()

    def reset(self):
        self.keys = [np.zeros((0, 0)) for _ in range(self.B)]
        self.toks = [np.zeros(0, dtype=np.int64) for _ in range(self.B)]
        self.pos = 0

    def step(self, h, y, theta, lam=0.0, row_loss=None, compute=True):
        """h [T,B,H] last-layer outputs (rounded to fp16 here), y [T,B] targets, theta >= 0, lam in [0, 1).
        row_loss [T*B] = -log p_model of every row (row n = t*B + b), or None.  Returns a dict with p_cache [T*B],
        empty [T*B] (no earlier position in the window: p_cache 0), and with row_loss also `row_loss` (mixed) and
        `loss` (summed over the batch, averaged over time).  compute=False only appends."""
        h = half_round(h)
        y = np.asarray(y, dtype=np.int64)
        T, B, H = h.shape
        assert B == self.B
        pc = np.zeros((T, B))
        empty = np.zeros((T, B), dtype=bool)
        for b in range(B):
            old = self.keys[b] if self.keys[b].size else np.zeros((0, H))
            K = np.concatenate([old, h[:, b]], axis=0)
            Y = np.concatenate([self.toks[b], y[:, b]])
            n_old = old.shape[0]
            if compute:
                j = np.arange(n_old + T)[None, :]
                qi = (n_old + np.arange(T))[:, None]
                ok = (j < qi) & (j >= qi - self.W)                 # C_t: the W positions before t, never t itself
                s = theta * (h[:, b] @ K.T)
                s = np.where(ok, s, -np.inf)
                m = s.max(axis=1, keepdims=True)
                has = np.isfinite(m[:, 0])
                e = np.where(ok, np.exp(s - np.where(np.isfinite(m), m, 0.0)), 0.0)
                match = Y[None, :] == y[:, b][:, None]
                num = (e * match).sum(axis=1)
                den = e.sum(axis=1)
                pc[:, b] = np.where(has, num / np.where(has, den, 1.0), 0.0)
                empty[:, b] = ~has
            self.keys[b] = K[-self.W:]
            self.toks[b] = Y[-self.W:]
        self.pos += T
        out = {"p_cache": pc.reshape(-1), "empty": empty.reshape(-1)}
        if row_loss is not None:
            rl = mix_row_loss(np.asarray(row_loss, dtype=np.float64).reshape(-1), out["p_cache"], out["empty"], lam)
            out["row_loss"] = rl
            out["loss"] = float(rl.mean() * B)
        return out
