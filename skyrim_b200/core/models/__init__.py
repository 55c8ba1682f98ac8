"""Model registry (reference: skyrim/core/models/__init__.py:9-17).  The H100 engine builds the
two step operators the north star names plus GraphCast (BASELINE config 4); the other reference wrappers
(fourcastnet, dlwp, fuxi, fengwu) are not part of this path."""
from .base import GlobalModel, GlobalPrediction, GlobalPredictionRollout  # noqa: F401
from .fourcastnet_v2 import FourcastnetV2Model
from .graphcast import GraphcastModel
from .pangu import PanguModel

MODELS = {"pangu": PanguModel, "fourcastnet_v2": FourcastnetV2Model, "graphcast": GraphcastModel}
