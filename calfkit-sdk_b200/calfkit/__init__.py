"""calfkit-b200: H100-native drop-in for the data-parallel hot path of calf-ai/calfkit-sdk.

Keeps the reference's public surface for that path (reference calfkit/__init__.py:10-30):
Client, Worker, Agent, agent_tool, ToolContext ... and puts a ctypes C-ABI over hand-written
sm_90a CUDA kernels underneath (see DESIGN.md)."""
__version__ = "0.1.0"

_LAZY = {
    "Client": ("calfkit.client", "Client"),
    "InvocationHandle": ("calfkit.client", "InvocationHandle"),
    "NodeResult": ("calfkit.client", "NodeResult"),
    "ToolContext": ("calfkit.models", "ToolContext"),
    "Agent": ("calfkit.nodes", "Agent"),
    "BaseNodeDef": ("calfkit.nodes", "BaseNodeDef"),
    "NodeDef": ("calfkit.nodes", "NodeDef"),
    "ToolNodeDef": ("calfkit.nodes", "ToolNodeDef"),
    "agent_tool": ("calfkit.nodes", "agent_tool"),
    "Worker": ("calfkit.worker", "Worker"),
}
__all__ = ["__version__", *_LAZY]


def __getattr__(name):
    if name in _LAZY:
        import importlib
        mod, attr = _LAZY[name]
        return getattr(importlib.import_module(mod), attr)
    raise AttributeError(name)
