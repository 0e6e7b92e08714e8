"""numpy fp32 restatement of iterate averaging (DESIGN.md section 16).

Averaging starts with n = 0.  Every averaged update sets n = n + 1 and, over the new weights theta:
    n = 1:  a = theta (a copy)
    n > 1:  a = a + ((theta - a) * mu),  mu = float32(1 / n) rounded once from double,
in fp32, each operation rounded on its own (numpy float32 arithmetic contracts nothing).
"""
import numpy as np


def mu(n):
    return np.float32(1.0 / float(n))


def avg_update(a, theta, n):
    """The average after update number n (>= 1) produced `theta` (fp32 arrays of one shape)."""
    theta = np.asarray(theta, dtype=np.float32)
    if n == 1:
        return theta.copy()
    a = np.asarray(a, dtype=np.float32)
    return (a + (theta - a) * mu(n)).astype(np.float32)


class Averager:
    """The n bookkeeping: start() restarts at n = 0 without touching the average; update(theta) averages one step."""

    def __init__(self):
        self.n, self.a = 0, None

    def start(self):
        self.n = 0

    def update(self, theta):
        self.n += 1
        self.a = avg_update(self.a, theta, self.n)
        return self.a
