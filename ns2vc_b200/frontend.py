"""Feature-side helper of the CLI / dataset path in front of the condition encoders (SURVEY.md §8(f) rank 4, first piece):
``repeat_expand_2d`` - the nearest-frame stretch of the ContentVec features [h, t_src] to the f0 frame count
(reference ``utils.py:482-496``, called from ``inference/infer_tool.py:166`` and ``dataset.py:37, 85``).

The reference walks the target frames in a Python loop and copies one column per iteration (on a CUDA tensor: one tiny kernel per
frame - about a thousand launches per slice, the same order as this package's whole first-call overhead for a new shape).  Here the
SAME walk runs on the host over the same fp32 boundary table and produces an index vector; the copy is one gather.  Bit-identical
output (``tests/test_frontend.py``, against outputs recorded from the reference's own function).

Drop-in: ``utils.repeat_expand_2d = ns2vc_b200.frontend.repeat_expand_2d`` after ``import utils``.
"""
from __future__ import annotations

from typing import List

import torch


def repeat_expand_index(src_len: int, target_len: int) -> List[int]:
    """Source column of every target column, exactly as the reference's walk chooses it: boundaries ``temp[j] = j * target_len /
    src_len`` in fp32 (int64 arange times int, true-divided: torch promotes to the default float dtype), the cursor advances by at
    most ONE column per target frame (so a down-stretch lags, like the reference)."""
    if src_len < 1 or target_len < 0:
        raise ValueError(f"repeat_expand: bad lengths {src_len} -> {target_len}")
    temp = (torch.arange(src_len + 1) * target_len / src_len).tolist()      # the reference's own expression (utils.py:487), fp32 values
    idx, pos = [], 0
    for i in range(target_len):
        if not (i < temp[pos + 1]):
            pos += 1
        idx.append(pos)
    return idx


def repeat_expand_2d(content: torch.Tensor, target_len: int) -> torch.Tensor:
    """content [h, t_src] -> float32 [h, target_len] on content's device (reference utils.py:482-496)."""
    if content.dim() != 2:
        raise ValueError(f"content must be [h, t], got {tuple(content.shape)}")
    idx = torch.tensor(repeat_expand_index(content.shape[-1], int(target_len)), dtype=torch.int64, device=content.device)
    return content.to(torch.float).index_select(1, idx)
