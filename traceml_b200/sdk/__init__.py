"""Public SDK surface (mirror of ``src/traceml/api.py:11-135``)."""
from .initial import TraceMLInitConfig, get_init_config, init, is_initialized, start
from .instrumentation import TraceState, trace_graph, trace_model_instance, trace_step, trace_time
from .wrappers import wrap_backward, wrap_dataloader_fetch, wrap_forward, wrap_h2d, wrap_optimizer

__all__ = ["TraceMLInitConfig", "init", "start", "get_init_config", "is_initialized", "trace_step",
           "trace_graph", "trace_time", "trace_model_instance", "TraceState", "wrap_dataloader_fetch",
           "wrap_forward", "wrap_backward", "wrap_optimizer", "wrap_h2d"]
