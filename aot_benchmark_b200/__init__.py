"""aot_benchmark_b200 -- H100-native AOT/DeAOT mask-propagation hot path.

Public surface (mirrors the reference's seam, SURVEY 8b):
    build_vos_model(name, cfg)            networks/models/__init__.py:5-11
    build_engine(name, phase, **kw)       networks/engines/__init__.py:5-21
    EngineConfig(exp, model)              configs/default.py:5-9
    TTAInferEngine(aot_model, ...)        networks/managers/evaluator.py:265-446 with TEST_FLIP / TEST_MULTISCALE
    MultiVideoInferEngine(aot_model, ...) several independent videos propagated in one batched pass per frame
    DeAOTMultiVideoInferEngine(...)       the same for the DeAOT models
    MultiVideoTTAInferEngine(...)         TTAInferEngine over several videos, one batched pass per scale per frame
"""
from .configs import EngineConfig  # noqa: F401
from .model import build_vos_model  # noqa: F401


def build_engine(name, phase="train", **kwargs):
    from .engine import build_engine as _b
    return _b(name, phase=phase, **kwargs)


def __getattr__(name):
    if name == "TTAInferEngine":          # imported on first use, like the engines behind build_engine
        from .tta import TTAInferEngine
        return TTAInferEngine
    if name in ("MultiVideoInferEngine", "DeAOTMultiVideoInferEngine"):
        from . import multi_video
        return getattr(multi_video, name)
    if name == "MultiVideoTTAInferEngine":
        from .multi_video_tta import MultiVideoTTAInferEngine
        return MultiVideoTTAInferEngine
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
