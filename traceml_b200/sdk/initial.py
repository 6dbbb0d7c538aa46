"""``traceml.init()`` policy (mirror of ``src/traceml/sdk/initial.py:55-276``).

Same modes, same validation messages' meaning, same idempotence / conflict
rules; installing patches additionally requires the CUDA engine to load, so a
missing extension or GPU fails here, loudly, not in the middle of training.
"""
from __future__ import annotations

from dataclasses import dataclass
from threading import Lock
from typing import Optional

_PATCH_FIELDS = ("patch_dataloader", "patch_forward", "patch_backward", "patch_h2d")


@dataclass(frozen=True)
class TraceMLInitConfig:
    mode: str
    patch_dataloader: bool
    patch_forward: bool
    patch_backward: bool
    patch_h2d: bool
    source: str = "user"

    def same_effective_configuration(self, other: "TraceMLInitConfig") -> bool:
        return self.mode == other.mode and all(
            getattr(self, f) == getattr(other, f) for f in _PATCH_FIELDS)


_LOCK = Lock()
_CONFIG: Optional[TraceMLInitConfig] = None


def _mode(mode: str) -> str:
    text = str(mode or "").strip().lower()
    if text == "custom":
        return "selective"
    if text in ("auto", "manual", "selective"):
        return text
    raise ValueError(
        f"Invalid TraceML init mode {mode!r}. Expected one of: 'auto', 'manual', 'selective'. "
        "The alias 'custom' is also accepted and maps to 'selective'.")


def _build(mode, overrides, source) -> TraceMLInitConfig:
    m = _mode(mode)
    given = {k: v for k, v in overrides.items() if v is not None}
    if m in ("auto", "manual"):
        if given:
            raise ValueError(
                "patch_dataloader, patch_forward, patch_backward, and patch_h2d may only be "
                f"provided when mode='selective'. Received overrides with mode={m!r}.")
        on = m == "auto"
        return TraceMLInitConfig(m, on, on, on, on, source)
    if not given:
        raise ValueError("mode='selective' requires at least one explicit patch_* override. "
                         "Use mode='manual' for no automatic patches.")
    vals = {f: bool(overrides.get(f)) for f in _PATCH_FIELDS}
    if not any(vals.values()):
        raise ValueError("mode='selective' must enable at least one automatic patch. "
                         "Use mode='manual' when you want zero automatic patches.")
    return TraceMLInitConfig("selective", source=source, **vals)


def _require_engine() -> None:
    """Fail at init, loudly, when the native engine cannot run here."""
    from .. import _abi

    _abi.lib()  # ImportError if libtraceml_b200.so is missing or stale
    import torch

    if not torch.cuda.is_available():
        raise RuntimeError(
            "traceml_b200.init(): no CUDA device is visible. The GPU-native engine records "
            "through CUDA kernels and has no CPU fallback; set TRACEML_DISABLED=1 to run untraced.")


def _apply(cfg: TraceMLInitConfig) -> None:
    from ..runtime import disabled

    if not disabled():
        _require_engine()
    if not any(getattr(cfg, f) for f in _PATCH_FIELDS):
        return
    try:
        from ..instrumentation import patches

        if cfg.patch_dataloader:
            patches.patch_dataloader()
        if cfg.patch_forward:
            patches.patch_forward()
        if cfg.patch_backward:
            patches.patch_backward()
        if cfg.patch_h2d:
            patches.patch_h2d()
    except Exception as exc:
        raise RuntimeError(
            "TraceML initialization failed while installing automatic instrumentation patches "
            f"for mode={cfg.mode!r}. This error is fatal because partial patch installation can "
            f"lead to inconsistent tracing behavior. Original error: {exc}") from exc


def get_init_config() -> Optional[TraceMLInitConfig]:
    return _CONFIG


def is_initialized() -> bool:
    return _CONFIG is not None


def init(*, mode: str = "auto", patch_dataloader: Optional[bool] = None,
         patch_forward: Optional[bool] = None, patch_backward: Optional[bool] = None,
         patch_h2d: Optional[bool] = None, _source: str = "user") -> TraceMLInitConfig:
    global _CONFIG
    req = _build(mode, {"patch_dataloader": patch_dataloader, "patch_forward": patch_forward,
                        "patch_backward": patch_backward, "patch_h2d": patch_h2d}, _source)
    with _LOCK:
        if _CONFIG is not None:
            if _CONFIG.same_effective_configuration(req):
                return _CONFIG
            raise RuntimeError(
                "TraceML has already been initialized with a different configuration in this "
                f"process. Existing config: {_CONFIG}. Requested config: {req}. Initialize "
                "TraceML exactly once per process with the intended mode at the start of the run.")
        _apply(req)
        _CONFIG = req
        return req


def enable_legacy_decorator_auto_init() -> Optional[TraceMLInitConfig]:
    """Importing the legacy decorator module used to install the automatic patches as a side
    effect (sdk/initial.py:303-317); an explicit ``init()`` made earlier is respected."""
    if is_initialized():
        return get_init_config()
    return init(mode="auto", _source="traceml.decorators")


def start(**kwargs) -> TraceMLInitConfig:
    return init(**kwargs)


def _reset_for_tests() -> None:
    global _CONFIG
    with _LOCK:
        _CONFIG = None


__all__ = ["enable_legacy_decorator_auto_init", "TraceMLInitConfig", "init", "start", "get_init_config", "is_initialized"]
