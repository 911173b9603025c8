"""llms — Python host-side mirror of the reference's LLM seam (reference pkg/llms/openai.go).

``LocalCUDAClient.Chat(model, max_tokens, prompts) -> str`` has the signature, return value and error
behaviour of ``(*OpenAIClient).Chat`` (openai.go:69-104); instead of POSTing to a remote
/chat/completions it calls the in-process sm_90a engine through the C ABI.  The Go binding a
maintainer would add is shown in INTEGRATION.md (Go is not available in this image).

Behaviour kept from the reference:
  * NewOpenAIClient rejects an empty apiKey with "OPENAI_API_KEY is not set"       (openai.go:40-42);
    the local provider accepts and ignores any non-empty key.
  * Retries = 5, Backoff = 1 s doubling after every 429/500                          (openai.go:57-60,91-94)
  * 401 -> fail at once; 429/500 -> sleep + retry; anything else -> fail at once     (openai.go:85-101)
  * after the last retry: "OpenAI request throttled after retrying 5 times"          (openai.go:103)
  * temperature = math.SmallestNonzeroFloat32 (greedy)                               (openai.go:73)
  * the result is Choices[0].Message.Content                                         (openai.go:82)
"""
from __future__ import annotations

import time
from dataclasses import dataclass

from .engine import Engine, EngineError

ChatMessageRoleSystem, ChatMessageRoleUser, ChatMessageRoleAssistant = "system", "user", "assistant"


@dataclass
class ChatCompletionMessage:        # go-openai ChatCompletionMessage{Role, Content}
    Role: str
    Content: str


class APIError(Exception):          # go-openai *APIError{HTTPStatusCode, Message}
    def __init__(self, status: int, message: str):
        super().__init__(f"error, status code: {status}, message: {message}")
        self.HTTPStatusCode, self.Message = status, message


class LocalCUDAClient:
    """Drop-in for llms.OpenAIClient: same fields (Retries, Backoff), same Chat()."""

    def __init__(self, engine: Engine, retries: int = 5, backoff: float = 1.0, sleep=time.sleep):
        self.engine, self.Retries, self.Backoff, self._sleep = engine, retries, backoff, sleep

    def _create_chat_completion(self, model: str, max_tokens: int, prompts) -> str:
        msgs = [(m.Role, m.Content) if isinstance(m, ChatCompletionMessage) else (m["role"], m["content"]) for m in prompts]
        try:
            return self.engine.chat_complete(model, msgs, max_tokens).content.decode("utf-8", "replace")
        except EngineError as e:
            raise APIError(e.code, e.message) from None

    def Chat(self, model: str, maxTokens: int, prompts) -> str:
        backoff = self.Backoff
        for _try in range(self.Retries):
            try:
                return self._create_chat_completion(model, maxTokens, prompts)
            except APIError as e:
                if e.HTTPStatusCode == 401:
                    raise
                if e.HTTPStatusCode in (429, 500):
                    self._sleep(backoff)
                    backoff *= 2
                    continue
                raise
        raise RuntimeError(f"OpenAI request throttled after retrying {self.Retries} times")


# unicode.IsSpace, the set strings.TrimSpace strips: Python's str.strip() also strips \x1c-\x1f, which Go keeps
GO_SPACE = "\t\n\v\f\r \x85\xa0\u1680\u2000\u2001\u2002\u2003\u2004\u2005\u2006\u2007\u2008\u2009\u200a\u2028\u2029\u202f\u205f\u3000"


def TrimSpace(s: str) -> str:
    """strings.TrimSpace"""
    return s.strip(GO_SPACE)


def NumTokensFromMessages(messages, model, count_tokens=None) -> int:
    """Mirror of pkg/llms/tokens.go:60.  For OpenAI names the reference counts with tiktoken; for local models it logs an error and
    returns 0 (tokens.go:61-66), which silently disables truncation.  Here the count comes from the engine's own tokenizer + chat
    template (`count_tokens` = Engine.count_tokens), so it is exact for the model that will read the prompt."""
    if count_tokens is None:
        return 0
    return int(count_tokens([(getattr(m, "Role", "") or "", getattr(m, "Content", "") or "") for m in messages]))


def ConstrictPrompt(prompt: str, model: str, tokenLimits: int, count_tokens=None) -> str:
    """Mirror of pkg/llms/tokens.go:128-144: while the prompt does not fit, drop its first ceil(n/3) lines."""
    import math
    while True:
        if NumTokensFromMessages([ChatCompletionMessage("", prompt)], model, count_tokens) < tokenLimits:
            return prompt
        lines = prompt.split("\n")
        lines = lines[int(math.ceil(len(lines) / 3)):]
        prompt = "\n".join(lines)
        if TrimSpace(prompt) == "":
            return ""


# pkg/llms/tokens.go:26-46: context windows by OpenAI model name (the reference's lookup data; lower-cased key, 4096 when unknown: tokens.go:49-56)
tokenLimitsPerModel = {"code-davinci-002": 4096, "gpt-3.5-turbo-0301": 4096, "gpt-3.5-turbo-0613": 4096, "gpt-3.5-turbo-1106": 16385, "gpt-3.5-turbo-16k-0613": 16385,
                       "gpt-3.5-turbo-16k": 16385, "gpt-3.5-turbo-instruct": 4096, "gpt-3.5-turbo": 4096, "gpt-4-0314": 8192, "gpt-4-0613": 8192, "gpt-4-1106-preview": 128000,
                       "gpt-4-32k-0314": 32768, "gpt-4-32k-0613": 32768, "gpt-4-32k": 32768, "gpt-4-vision-preview": 128000, "gpt-4": 8192, "text-davinci-002": 4096,
                       "text-davinci-003": 4096, "qwen-plus": 4096}


def GetTokenLimits(model: str, engine_limit: int | None = None) -> int:
    """Mirror of pkg/llms/tokens.go:49-56.  `engine_limit` (the local engine's max_seq_len, Engine.info["max_seq_len"]) wins when given: the engine
    answers to any model name (model_aliases "*"), and what bounds a request is ITS context window, not the window of the name the caller sent."""
    if engine_limit:
        return int(engine_limit)
    return tokenLimitsPerModel.get(model.lower(), 4096)


def ConstrictMessages(messages, model: str, maxTokens: int, count_tokens=None, engine_limit: int | None = None):
    """Mirror of pkg/llms/tokens.go:110-125: None when maxTokens alone exceeds the window; otherwise drop the oldest message after the first (the
    system prompt) until prompt + maxTokens fit.  The reference slices messages[2:] unconditionally, so a single message that does not fit panics
    there (slice bounds out of range); here that case raises IndexError with the same meaning.  (No caller in the reference uses it today —
    AssistantWithConfig truncates observations with ConstrictPrompt instead — it is mirrored because it is part of the pkg/llms surface.)"""
    tokenLimits = GetTokenLimits(model, engine_limit)
    if maxTokens >= tokenLimits:
        return None
    messages = list(messages)
    while True:
        if NumTokensFromMessages(messages, model, count_tokens) + maxTokens < tokenLimits:
            return messages
        if len(messages) < 2:
            raise IndexError("slice bounds out of range [2:%d]" % len(messages))
        messages = messages[:1] + messages[2:]


_ENGINES: dict = {}


def new_client(api_key: str, base_url: str, engine: Engine | None = None, engine_config: dict | None = None) -> LocalCUDAClient:
    """Mirror of NewOpenAIClient(apiKey, baseURL).  base_url ``cuda://<model>`` (or an explicit engine)
    selects the local provider; the engine handle is a process singleton per base_url because the
    reference constructs a client per request (pkg/assistants/simple.go:316)."""
    if api_key == "":
        raise ValueError("OPENAI_API_KEY is not set")
    if engine is None:
        if not base_url.startswith("cuda://"):
            raise ValueError("only the local-cuda provider is implemented here: base_url must be cuda://<model>")
        if base_url not in _ENGINES:
            cfg = dict(engine_config or {})
            cfg.setdefault("model", base_url[len("cuda://"):])
            _ENGINES[base_url] = Engine(cfg)
        engine = _ENGINES[base_url]
    return LocalCUDAClient(engine)
