"""Dynamic evaluation (Krause, Kahembwe, Murray & Renals, "Dynamic Evaluation of Neural Sequence Models", ICML 2018;
DESIGN.md section 14): score the text one window at a time and, after each window, take a gradient step on it, pulled
back toward the trained weights theta_g.  Driven through `Trainer.gradient_stats`, `Trainer.dynamic_eval_step` and
`Trainer.dynamic_perplexity`; this module holds the gradient statistics of the RMS rule.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch


@dataclass
class GradStats:
    """The RMS rule's statistics (zrb_grad_stats_step / _finish) over `windows` gradient windows at theta_g.

    rms:  flat fp32 CUDA tensor in the Trainer's flat layout (a tied E next to fc.b): r = sqrt(mean of g^2) per element
    mean: 0-d fp32 CUDA tensor, r-bar = the mean of r over all parameter elements (fixed-order fp64 sum, rounded once)
    """
    rms: torch.Tensor
    mean: torch.Tensor
    windows: int
