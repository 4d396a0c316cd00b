"""The one place that decides whether the caller allowed TF32 matmuls.

torch has two ways to allow them: the legacy ``torch.backends.cuda.matmul.allow_tf32`` /
``torch.set_float32_matmul_precision("high")``, and the newer ``fp32_precision`` attributes
(``torch.backends.cuda.matmul.fp32_precision = "tf32"`` or ``torch.backends.fp32_precision = "tf32"``).  Once the newer
API has been used, reading ``allow_tf32`` raises ("mix of the legacy and new APIs"); reading
``torch.backends.cuda.matmul.fp32_precision`` works after any of the four setters and disturbs no later legacy read.
"""
from __future__ import annotations

import torch


def tf32_allowed() -> bool:
    """True when torch allows TF32 for fp32 CUDA matmuls, through either API."""
    return torch.backends.cuda.matmul.fp32_precision == "tf32"
