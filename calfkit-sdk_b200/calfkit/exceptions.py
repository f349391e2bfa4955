class DeserializationError(Exception):
    """Raised client-side when the expected output part is missing from a reply
    (mirrors reference calfkit/exceptions.py; raised from client/deserialize.py:72,80,89)."""


class EngineError(RuntimeError):
    """The GPU batch engine reported a failure (missing CUDA library, CUDA error, ...).
    There is no CPU fallback: the engine fails loudly instead."""


class RecordRejected(ValueError):
    """A single record failed device-side validation; carries the pydantic-style error class."""

    def __init__(self, status: int, name: str, index: int):
        super().__init__(f"record {index}: {name} (status {status})")
        self.status = status
        self.name = name
        self.index = index
