"""skyrim_b200 — H100-native rollout engine behind the Skyrim API (see DESIGN.md)."""
__all__ = ["Skyrim"]


def __getattr__(name):
    if name == "Skyrim":
        from .core.skyrim import Skyrim
        return Skyrim
    raise AttributeError(name)
