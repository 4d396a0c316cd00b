"""The one place that decides whether the caller asked for deterministic algorithms, and PyTorch's alert for an op that
has no deterministic implementation.

``torch.use_deterministic_algorithms(True)`` asks every op to either run a deterministic implementation or raise
(``warn_only=True``: warn instead).  torch has no Python-level form of its internal alert, so ``alert_not_deterministic``
restates it with torch's message.
"""
from __future__ import annotations

import warnings

import torch


def deterministic_requested() -> bool:
    """True under ``torch.use_deterministic_algorithms(True)`` (with or without ``warn_only``)."""
    return torch.are_deterministic_algorithms_enabled()


def alert_not_deterministic(caller: str) -> None:
    """Raise RuntimeError (or warn under ``warn_only=True``) when determinism is requested; no-op otherwise."""
    if not deterministic_requested():
        return
    msg = (f"{caller} does not have a deterministic implementation, but you set "
           "'torch.use_deterministic_algorithms(True)'. You can turn off determinism just for this operation, or you "
           "can use the 'warn_only=True' option, if that's acceptable for your application.")
    if torch.is_deterministic_algorithms_warn_only_enabled():
        warnings.warn(msg, UserWarning, stacklevel=3)
    else:
        raise RuntimeError(msg)
