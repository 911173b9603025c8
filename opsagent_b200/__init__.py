"""opsagent_b200 — H100-native local chat-completion engine behind OpsAgent's pkg/llms seam.

Python host-side mirror of the reference interface for the hot path:
  llms.LocalCUDAClient.Chat(model, max_tokens, prompts)  <->  reference pkg/llms/openai.go:69
  assistants.AssistantWithConfig(...)                    <->  reference pkg/assistants/simple.go:292
The compute lives in lib/libopsagent_b200.so (hand-written sm_90a CUDA; C ABI in include/opsagent_b200.h).
"""
from . import _lib  # noqa: F401
from .engine import Engine, EngineError  # noqa: F401
from .llms import LocalCUDAClient, APIError, ChatCompletionMessage, new_client  # noqa: F401

__all__ = ["Engine", "EngineError", "LocalCUDAClient", "APIError", "ChatCompletionMessage", "new_client"]
