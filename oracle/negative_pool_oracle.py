"""TEST INFRASTRUCTURE ONLY -- the reference solver's negative pool restated on the host, line for line.

bm/solver.py cannot be imported without flashy, dora, hydra, julius and mne.  `HostNegativePool` restates
`Solver._make_negative_pool` (bm/solver.py:152-164) and the negatives block of `Solver._run_one_epoch`
(bm/solver.py:358-371): one CPU tensor per phase, `torch.randperm` on the CPU default generator, `torch.cat` of the batch
and the drawn rows under `torch.no_grad()`, and the new pool `[output; buf[kept]; old buf][:negative_pool_size]`.  The
fixture generator (`oracle/make_negative_pool_golden.py`) and the GPU tests feed its candidates to a ClipLoss.
"""
from __future__ import annotations

import typing as tp

import torch


class HostNegativePool:
    def __init__(self, negatives: tp.Optional[int], negative_pool_size: tp.Optional[int] = None):
        # solver.py:152-159
        if negatives is not None:
            if negative_pool_size is None:
                negative_pool_size = 2 * negatives
            assert negative_pool_size >= negatives, \
                "Pool of negatives should be larger than the number of negatives"
        self.negatives = negatives
        self.negative_pool_size = negative_pool_size
        # solver.py:161-163
        self.negative_pool = {name: torch.Tensor([], device="cpu") for name in ["train", "valid"]}
        self.last_kept: tp.Optional[torch.Tensor] = None     # the draw of the last pooled call (None: no pool code ran)

    def complete(self, output: torch.Tensor, training: bool) -> torch.Tensor:
        """solver.py:358-371: the candidates the loss receives"""
        self.last_kept = None
        with torch.no_grad():
            n_negatives = self.negatives
            if n_negatives is not None:
                if len(output) < n_negatives:
                    phase = 'train' if training else 'valid'
                    buf = self.negative_pool[phase]
                    n_kept = n_negatives - len(output)
                    kept = torch.randperm(len(buf))[:n_kept]
                    self.last_kept = kept
                    output = torch.cat([output, buf[kept].to(output.device)], dim=0)
                    buf = torch.cat([output.to(buf.device), buf])
                    self.negative_pool[phase] = buf[:self.negative_pool_size]
        return output
