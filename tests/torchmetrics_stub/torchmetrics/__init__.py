"""Stand-in for the surface of torchmetrics 0.7 that the reference's metric classes (model_training/metrics) and
FlameLightningModel (MetricCollection) touch: ``Metric`` with ``add_state`` / ``reset`` / ``forward`` and the
``update`` / ``compute`` wrapping, and ``MetricCollection``.  torchmetrics is not installed here; the semantics below are
restated from the 0.7 release's ``torchmetrics/metric.py`` and ``collections.py`` as read, not run against that release:
- ``forward(*args)`` (compute_on_step=True): update the accumulated state with the batch; then, on a fresh state, update
  with the batch alone, take ``compute()`` as the value to return, and restore the accumulated state.  With
  compute_on_step=False it only updates and returns None.
- ``compute()`` returns its cached value until the next ``update``; ``reset()`` restores the defaults.
- States are tensors (``dist_reduce_fx`` is recorded; there is no distributed sync here).
TEST INFRASTRUCTURE ONLY: put ``tests/torchmetrics_stub`` on sys.path to use it."""
from __future__ import annotations

import copy
import functools
from typing import Any, Callable, Dict, Optional

import torch
from torch import nn

__version__ = "0.7.0"
__all__ = ["Metric", "MetricCollection"]


class Metric(nn.Module):
    def __init__(self, compute_on_step: bool = True, dist_sync_on_step: bool = False, process_group: Optional[Any] = None,
                 dist_sync_fn: Callable = None):
        super().__init__()
        self.compute_on_step = compute_on_step
        self.dist_sync_on_step = dist_sync_on_step
        self.process_group = process_group
        self.dist_sync_fn = dist_sync_fn
        self._defaults: Dict[str, torch.Tensor] = {}
        self._reductions: Dict[str, Any] = {}
        self._computed = None
        self._forward_cache = None
        self._update_called = False
        self.update = self._wrap_update(self.update)
        self.compute = self._wrap_compute(self.compute)

    def add_state(self, name: str, default, dist_reduce_fx=None, persistent: bool = False):
        if not isinstance(default, torch.Tensor):
            raise ValueError("the stand-in only holds tensor states")
        setattr(self, name, default.clone())
        self._defaults[name] = default.detach().clone()
        self._reductions[name] = dist_reduce_fx

    def _wrap_update(self, update):
        @functools.wraps(update)
        def wrapped(*args, **kwargs):
            self._computed = None
            self._update_called = True
            return update(*args, **kwargs)
        return wrapped

    def _wrap_compute(self, compute):
        @functools.wraps(compute)
        def wrapped(*args, **kwargs):
            if self._computed is None:
                self._computed = compute(*args, **kwargs)
            return self._computed
        return wrapped

    def _state(self):
        return {k: getattr(self, k) for k in self._defaults}

    def forward(self, *args, **kwargs):
        self.update(*args, **kwargs)
        if not self.compute_on_step:
            return None
        cache = {k: v.clone() for k, v in self._state().items()}
        self.reset()
        self.update(*args, **kwargs)
        self._forward_cache = self.compute()
        for k, v in cache.items():
            setattr(self, k, v)
        self._computed = None
        self._update_called = True
        return self._forward_cache

    def reset(self):
        self._update_called = False
        self._forward_cache = None
        self._computed = None
        for k, v in self._defaults.items():
            setattr(self, k, v.detach().clone().to(getattr(self, k).device))

    def update(self, *args, **kwargs):  # overridden
        raise NotImplementedError

    def compute(self):  # overridden
        raise NotImplementedError


class MetricCollection(nn.ModuleDict):
    """A dict of metrics called together: ``forward`` / ``compute`` return {name: value} in insertion order."""

    def __init__(self, metrics, prefix: Optional[str] = None, postfix: Optional[str] = None):
        super().__init__()
        if isinstance(metrics, (list, tuple)):
            metrics = {type(m).__name__: m for m in metrics}
        for name, m in metrics.items():
            if not isinstance(m, Metric):
                raise ValueError(f"value {m} belonging to key {name} is not an instance of torchmetrics.Metric")
            self[name] = m
        self.prefix, self.postfix = prefix or "", postfix or ""

    def _key(self, k):
        return f"{self.prefix}{k}{self.postfix}"

    def forward(self, *args, **kwargs):
        return {self._key(k): m(*args, **kwargs) for k, m in self.items()}

    def update(self, *args, **kwargs):
        for m in self.values():
            m.update(*args, **kwargs)

    def compute(self):
        return {self._key(k): m.compute() for k, m in self.items()}

    def reset(self):
        for m in self.values():
            m.reset()

    def clone(self):
        return copy.deepcopy(self)
