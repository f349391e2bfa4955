"""CPU test of the walker's id-keyed dicts (tool_calls / tool_results) across sizes: the thread walker keeps the first
few keys in registers and re-scans the dict for the later ones (ck_walk.cuh DictKeys).  Dicts of up to 128 entries
(CK_DICT_KEYS) stay on the fast path, duplicates are rejected wherever they sit, and tool_calls[input_args[0]] /
tool_results[input_args[0]] resolve to the right entry whatever its index."""
import pytest

from calfkit import synth
from calfkit.engine._lib import COL
from hostsim import walk, walk_global
from pydantic import ValidationError

TS = synth.TS


def _record(keys: list[str], pick: str, n_results: int | None = None) -> tuple[bytes, dict, dict]:
    calls = {k: synth.tool_call_part(f"tool_{i:03d}", '{"location":%s}' % synth.jstr(f"city {i}"), k) for i, k in enumerate(keys)}
    results = {k: '{"v":%d}' % i for i, k in enumerate(keys[:len(keys) if n_results is None else n_results])}
    frames = [synth.frame("agent.input", "calf-client-reply-00", None, "f0"),
              synth.frame("tool.x.input", "agent.input", [pick, "agent"], "f1")]
    rec = synth.envelope(tool_calls=calls, tool_results=results, uncommitted="null", history=[synth.user_request("hi")],
                         final_parts=[], temp_instructions=None, state_metadata="null", state_overrides="null",
                         correlation_id="c0", provided_deps="{}", frames=frames)
    return rec.encode(), calls, results


def _dup_record(keys: list[str]) -> bytes:
    # a dict literal cannot hold a duplicate: splice the entries by hand
    rec, calls, _ = _record(keys[:1], keys[0], 0)
    body = ",".join(synth.jstr(k) + ":" + calls[keys[0]].replace(keys[0], k) for k in keys)
    one = synth.jstr(keys[0]) + ":" + calls[keys[0]]
    return rec.replace(one.encode(), body.encode(), 1)


def _is_fixed(b: bytes) -> bool:
    from calfkit.models import Envelope
    try:
        return Envelope.model_validate_json(b).model_dump_json().encode() == b
    except ValidationError:
        return False


def _span(b: bytes, cols, name: str) -> bytes:
    off, ln = int(cols[COL[name + "_OFF"]]), int(cols[COL[name + "_LEN"]])
    return b[off:off + ln]


@pytest.mark.parametrize("n", [1, 2, 3, 5, 17, 127, 128])
def test_dict_sizes_resolve_every_index(n):
    keys = [f"call_{i:05d}x" for i in range(n)]
    for j in sorted({0, 1, 2, n // 2, n - 1} & set(range(n))):
        for n_res in (n, 0, j + 1):
            b, calls, results = _record(keys, keys[j], n_res)
            acc, cols = walk(b)
            assert acc, (n, j, n_res)
            if n <= 5:
                assert _is_fixed(b)
            assert _span(b, cols, "CALL_VAL") == calls[keys[j]].encode(), (n, j)
            assert _span(b, cols, "TNAME") == synth.jstr(f"tool_{j:03d}").encode()[1:-1]
            assert _span(b, cols, "RES") == (results[keys[j]].encode() if keys[j] in results else b""), (n, j, n_res)
            acc_g, cols_g = walk_global(b)      # the global-load reader: the same verdict and columns
            assert acc_g and (cols == cols_g).all()
    b, _, _ = _record(keys, "call_none", n)  # a key that is not in the dicts
    acc, cols = walk(b)
    assert acc and _span(b, cols, "CALL_VAL") == b"" and _span(b, cols, "RES") == b""


def test_more_than_128_entries_leave_the_fast_path():
    keys = [f"call_{i:05d}x" for i in range(129)]
    b, _, _ = _record(keys, keys[5], 0)
    assert not walk(b)[0]
    b, _, _ = _record(keys[:128], keys[5], 0)
    assert walk(b)[0]


@pytest.mark.parametrize("n,dup_of", [(2, 0), (3, 0), (3, 2), (40, 1), (40, 30), (128, 127), (128, 0)])
def test_duplicate_keys_are_rejected_at_any_index(n, dup_of):
    keys = [f"call_{i:05d}x" for i in range(n - 1)]
    keys.append(keys[dup_of] if dup_of < n - 1 else keys[0])
    b = _dup_record(keys)
    assert not walk(b)[0] and not walk_global(b)[0]
    assert not _is_fixed(b)
    keys[-1] = "call_uniq"
    assert walk(_dup_record(keys))[0]
