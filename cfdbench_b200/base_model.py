"""AutoCfdModel base class.

When the reference's `src/` directory is on sys.path (i.e. when `train_auto.py` / `test_multistep.py`
drive this package through `cfdbench_b200.runner`), the drop-in model must subclass the *reference's*
class, because `test_multistep.py:109` checks `isinstance(model, AutoCfdModel)`.  Stand-alone (tests,
bench, or wherever the reference is not importable) a mirror with the same three abstract
methods is used (reference src/models/base_model.py:41-81).
"""
from __future__ import annotations

from typing import List, Optional

from torch import Tensor, nn

try:  # pragma: no cover - only when the reference is importable
    from models.base_model import AutoCfdModel  # type: ignore
    USING_REFERENCE_BASE = True
except Exception:  # noqa: BLE001
    USING_REFERENCE_BASE = False

    class AutoCfdModel(nn.Module):  # type: ignore[no-redef]
        """A CFD model that generates the solution auto-regressively, one frame at a time."""

        def __init__(self, loss_fn: nn.Module):
            super().__init__()
            self.loss_fn = loss_fn

        def forward(self, inputs: Tensor, label: Optional[Tensor] = None, case_params: Optional[dict] = None,
                    mask: Optional[Tensor] = None, **kwargs) -> dict:
            raise NotImplementedError

        def generate(self, inputs: Tensor, case_params: Tensor, mask: Tensor, **kwargs) -> Tensor:
            raise NotImplementedError

        def generate_many(self, inputs: Tensor, case_params: Tensor, mask: Tensor, steps: int,
                          **kwargs) -> List[Tensor]:
            raise NotImplementedError
