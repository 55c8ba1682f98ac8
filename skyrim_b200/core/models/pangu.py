"""PanguModel — mirrors /root/reference/skyrim/core/models/pangu.py:17-62; ``build_model``
returns the CUDA TimeLoop instead of ``pangu.load(registry.get_model("e2mip://pangu"))``."""
from __future__ import annotations

from ...config import PANGU_CHANNELS, PanguConfig, pangu_full
from ...schedule import check_schedule
from .base import GlobalModel

CHANNELS = PANGU_CHANNELS


class PanguModel(GlobalModel):
    """``schedule="6h"`` (the default) chains the 6-h operator.  ``schedule="hierarchical"`` interleaves it with the 24-h
    operator as earth2mip's PanguInference does (``skyrim_b200/schedule.py``): still one slice every 6 h, the slice at
    24 d + 6 k hours being P6^k(P24^d(x0)); ``rollout(save=False)`` and ``predict`` then compute only their two slices,
    with the fewest forwards.  The 24-h operator's parameters are ``weights_24``, else those in the checkpoint directory
    ``SKYRIM_B200_WEIGHTS`` names (when ``weights`` is not given either), else the synthetic
    ``make_pangu_weights(cfg, weight_seed_24)``; its seed defaults to ``weight_seed + 1`` so that the two synthetic
    operators differ, as the real ones do."""
    model_name = "pangu"

    def __init__(self, *args, cfg: PanguConfig | None = None, weights=None, weight_seed: int = 0, device: int = 0,
                 schedule: str = "6h", weights_24=None, weight_seed_24: int | None = None, **kwargs):
        self.schedule = check_schedule(schedule)
        if schedule == "6h" and (weights_24 is not None or weight_seed_24 is not None):
            raise ValueError("weights_24 and weight_seed_24 belong to schedule='hierarchical'")
        self._cfg, self._weights, self._seed, self._device = cfg or pangu_full(), weights, weight_seed, device
        self._weights_24 = weights_24
        self._seed_24 = weight_seed + 1 if weight_seed_24 is None else weight_seed_24
        super().__init__(self.model_name, *args, **kwargs)

    def build_model(self):
        from ...engine import StepEngine
        from ...timeloop import PanguHierarchicalTimeLoop, PanguTimeLoop
        from ...weights import make_pangu_weights
        import os
        w, w24 = self._weights, self._weights_24
        real = os.environ.get("SKYRIM_B200_WEIGHTS")
        from_files = w is None and bool(real)
        if from_files:
            # real checkpoint on disk (what pangu.load(registry.get_model("e2mip://pangu")) downloads in the reference,
            # pangu.py:45-46): ONNX initialisers -> engine parameters, no onnx / onnxruntime needed (importers.py)
            from ...importers import load_pangu_pair, load_real_weights
            if self.schedule == "6h":
                _, w = load_real_weights("pangu", real)
            else:
                w, file_24 = load_pangu_pair(real, self._cfg)
                w24 = file_24 if w24 is None else w24
        eng = StepEngine(self._cfg, self._device)
        # no network here: without SKYRIM_B200_WEIGHTS or a weight dict the engine runs on seeded synthetic weights
        eng.load_weights(w if w is not None else make_pangu_weights(self._cfg, self._seed))
        if self.schedule == "6h":
            loop = PanguTimeLoop(eng)
        else:
            eng_24 = StepEngine(self._cfg, self._device)
            eng_24.load_weights(w24 if w24 is not None else make_pangu_weights(self._cfg, self._seed_24))
            loop = PanguHierarchicalTimeLoop(eng, eng_24)
        # a real checkpoint feeds un-normalised residual streams to fp16 tensor-core operands: the first step of every
        # rollout runs with the engine's fp16-range guard (StepEngine.step_guarded raises above 3e4)
        loop.guard_first_step = from_files
        return loop

    def release_model(self):
        if self.schedule == "hierarchical":
            self.model.engine_24.close()
        super().release_model()

    @property
    def device(self):
        return self.model.device
