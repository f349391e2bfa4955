"""Batched client reply path (SURVEY.md §8f row 3): what `deserialize_to_node_result(...).output` yields for every
reply of a batch (reference calfkit/client/deserialize.py:15-89 — first DataPart.data, else first TextPart.text;
`output_type=str` forces text; any other type validates DataPart.data) without building the Python object tree of
each envelope: the CUDA walker validates the replies and records the two candidate spans, `ck_reply_plan` selects
one per record, the emit kernel gathers the values, and the host only decodes that value's JSON (plus the
`TypeAdapter` validation the reference also runs on the host for typed outputs).

`InvocationHandle.result()` stays the per-request API (it needs message_history etc. as objects); this is the
throughput path for consumers that only want outputs keyed by correlation id."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any

import pydantic_core
from pydantic import TypeAdapter

from calfkit.broker import Record
from calfkit.client.deserialize import _UNSET
from calfkit.engine._lib import CK_ACT_REPLY, CK_OK, CK_SKIPPED, COL, STATUS_NAMES
from calfkit.exceptions import DeserializationError, RecordRejected
from calfkit.engine.lane import FetchArena
from calfkit.nodes.base import submit_inbound


@dataclass
class ReplyOutput:
    correlation_id: str | None
    output: Any = None
    error: Exception | None = None      # DeserializationError / pydantic ValidationError / RecordRejected, as the reference would raise


class BatchReplyDecoder:
    def __init__(self, engine):
        self.engine = engine

    def decode(self, records: list[Record] | list[bytes] | FetchArena, output_type: type[Any] = _UNSET) -> list[ReplyOutput]:
        """one ReplyOutput per delivered record, Records or the records of a fetch response alike"""
        if not isinstance(records, FetchArena):
            records = [r if isinstance(r, Record) else Record("", r, None, None) for r in records]
            if not records:
                return []
        eng = self.engine
        inb = submit_inbound(eng, records)
        mode = 0 if output_type is _UNSET else (1 if output_type is str else 2)
        eng.reply_plan(mode)
        out = eng.fetch()
        cols = out.cols
        adapter = TypeAdapter(output_type) if mode == 2 else None
        res: list[ReplyOutput] = []
        for i in range(inb.n):
            if cols[COL["STATUS"], i] == CK_SKIPPED:          # not delivered to a consumer (a control / aborted batch)
                continue
            if cols[COL["STATUS"], i] != CK_OK:
                st = int(cols[COL["STATUS"], i])
                res.append(ReplyOutput(inb.correlation_ids[i], error=RecordRejected(st, STATUS_NAMES[st], i)))
                continue
            rec = out.record_bytes(i)
            c0 = int(cols[COL["CORR_OFF"], i])
            corr = pydantic_core.from_json(b'"' + bytes(rec[c0:c0 + int(cols[COL["CORR_LEN"], i])]) + b'"')
            if cols[COL["ACTION"], i] != CK_ACT_REPLY:
                what = {0: "No DataPart or TextPart found in final_output_parts; cannot auto-detect output.",
                        1: "No TextPart found in final_output_parts; expected output_type=str.",
                        2: "No DataPart found in final_output_parts; expected output_type="
                           f"{getattr(output_type, '__name__', str(output_type))}."}[mode]
                res.append(ReplyOutput(corr, error=DeserializationError(what)))
                continue
            value = pydantic_core.from_json(out.payload(i))
            if adapter is not None:
                try:
                    value = adapter.validate_python(value)
                except Exception as e:  # noqa: BLE001  (pydantic ValidationError, as in the reference)
                    res.append(ReplyOutput(corr, error=e))
                    continue
            res.append(ReplyOutput(corr, output=value))
        return res
