"""The fetch's record split (ck_rb_split_kernel) and field decode (ck_rb_fields_kernel, csrc/ck_kafka.cuh) held record by
record against the strict reference parser (tests/kafka_records_ref.py), on record sets whose CRC32C is valid so that
every case reaches the parser: one hand-built case per parse rule, structured mutations of seeded batches packed by the
thousand into one fetch with an untouched batch between them, the same records inside each codec's simplest container,
and the host's batch chain.  Compared per record: the verdict, the value, key and correlation id bytes under the spans
rb_index() reports (and the offsets themselves for an uncompressed batch), no span on a refused record, and the status
column CK_BAD_FRAME exactly where the record is bad."""
import numpy as np
import pytest

import kafka_record_cases as kc
import kafka_records_ref as ref
import kafka_txn as kt

pytestmark = pytest.mark.gpu

MAX_RECORDS = 1 << 16


@pytest.fixture(scope="module")
def eng():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from calfkit.engine import BatchEngine, ToolTemplate
    e = BatchEngine(0, max_records=MAX_RECORDS, max_in_bytes=64 << 20)
    e.register_topics(["tool.get_weather.input", "tool.get_weather.output", "weather_agent.input"], num_partitions=8)
    e.set_tool_node("tool.get_weather.output", ToolTemplate.from_format("It's sunny in {location}"))
    yield e
    e.close()


def check(e, buf: bytes, labels: list[str]) -> None:
    """submit `buf` once; every record as the reference says.  labels[b]: the name of complete batch b, for the report"""
    from calfkit.engine._lib import CK_BAD_FRAME, COL
    want = ref.parse_fetch(buf, MAX_RECORDS)
    n = e.submit_recordbatch(np.frombuffer(buf, dtype=np.uint8))
    ix = e.fetch_index
    e.tool_plan()
    status = e.fetch().cols[COL["STATUS"]]
    assert n == len(want)
    owner = [labels[b] for b, (s, _e) in enumerate(kt.batches(buf)) for _ in range(int.from_bytes(buf[s + 57:s + 61], "big"))]
    d = ix["data"]
    fails = []
    for i, r in enumerate(want):
        vo, vl, ko, kl, co, cl = (int(ix[k][i]) for k in ("val_off", "val_len", "key_off", "key_len", "corr_off", "corr_len"))
        got = {"bad": int(ix["bad"][i]), "bad_frame_status": bool(status[i] == CK_BAD_FRAME)}
        exp = {"bad": r.bad, "bad_frame_status": r.bad == 1}
        if r.bad:
            got["spans"], exp["spans"] = (vo, vl, kl, cl), (0, 0, -1, -1)
        else:
            got["value"], exp["value"] = d[vo:vo + vl].tobytes(), r.value()
            got["key"], exp["key"] = (None if kl < 0 else d[ko:ko + kl].tobytes()), r.key_bytes()
            got["corr"], exp["corr"] = (None if cl < 0 else d[co:co + cl].tobytes()), r.corr_bytes()
            if not r.decoded:                                  # spans into the fetch itself: the offsets too
                got["offsets"] = (vo, vl, ko if kl >= 0 else None, co if cl >= 0 else None)
                exp["offsets"] = (*r.val, r.key and r.key[0], r.corr and r.corr[0])
        for k in exp:
            if got[k] != exp[k]:
                fails.append(f"record {i} of {owner[i]!r}: {k} {got[k]!r} != {exp[k]!r}")
    assert not fails, f"{len(fails)} mismatches:\n" + "\n".join(fails[:30])


def interleave(named: list[tuple[str, bytes]], filler: list[bytes]) -> tuple[bytes, list[str]]:
    """the batches with an untouched batch before each of them and one at the end"""
    parts, labels = [], []
    for k, (name, b) in enumerate(named):
        parts += [filler[k % len(filler)], b]
        labels += [f"untouched before {name}", name]
    parts.append(filler[0])
    labels.append("untouched at the end")
    return b"".join(parts), labels


HAND = kc.hand_cases()


@pytest.mark.parametrize("name", list(HAND))
def test_hand_case(eng, name):
    b, _verdict = HAND[name]
    good = kc.batch(kc.A + kc.B, 2)
    buf, labels = interleave([(name, b)], [good])
    check(eng, buf, labels)


def test_all_hand_cases_in_one_fetch(eng):
    buf, labels = interleave([(n, b) for n, (b, _v) in HAND.items()], kc.sources(11, 5))
    check(eng, buf, labels)


def test_every_varint_operator_at_every_varint(eng):
    srcs = kc.sources(21, 8)
    muts = kc.mutants(srcs)
    assert len(muts) > 1500
    for k in range(0, len(muts), 3000):
        check(eng, *interleave(muts[k:k + 3000], srcs))


@pytest.mark.parametrize("seed", [31, 32, 33])
def test_seeded_mutation_sample(eng, seed):
    srcs = kc.sources(seed, 40)
    muts = kc.mutants(srcs, exhaustive=False, sample=3000, seed=seed)
    check(eng, *interleave(muts, srcs[:5]))


@pytest.mark.parametrize("codec", sorted(kc.CONTAINERS), ids=lambda c: kc.CODEC_NAMES[c])
def test_decoded_slots_parse_as_the_uncompressed_sections(eng, codec):
    """hand cases and mutants inside the codec's container, between untouched uncompressed and compressed batches: the
    verdicts and span bytes the reference gives the uncompressed batches"""
    srcs = kc.sources(41, 6)
    named = [(n, b) for n, (b, _v) in HAND.items() if n not in kc.HEADER_CASES]
    named += kc.mutants(srcs, exhaustive=False, sample=400, seed=41 + codec)
    wrapped = [(f"{kc.CODEC_NAMES[codec]} {n}", kc.wrap(b, codec)) for n, b in named]
    for (_n, b), (_w, z) in zip(named, wrapped):
        plain, packed = ref.parse_fetch(b), ref.parse_fetch(z)
        assert [(r.bad, r.value(), r.key_bytes(), r.corr_bytes()) for r in plain] == \
            [(r.bad, r.value(), r.key_bytes(), r.corr_bytes()) for r in packed]
    check(eng, *interleave(wrapped, srcs + [kc.wrap(s, codec) for s in srcs]))


def test_short_batch_length_ends_the_chain(eng):
    """a batchLength below 49 ends the chain: the records before it are delivered, nothing after it is counted"""
    import struct
    good = kc.sources(51, 3)
    for blen in (48, 0, -1):
        buf = good[0] + good[1] + struct.pack(">qi", 0, blen) + b"\0" * 60 + good[2]
        assert len(kt.batches(buf)) == 2
        check(eng, buf, ["first", "second"])


def test_records_count_past_max_records_is_refused_and_the_engine_recovers(eng):
    """a batch whose CRC-covered recordsCount passes max_records refuses the whole fetch, naming max_records; the next
    valid fetch on the same engine decodes as the reference says"""
    from calfkit.exceptions import EngineError
    srcs = kc.sources(61, 4)
    for count in (MAX_RECORDS + 1, 0x7FFFFFFF, 0xFFFFFFFF):
        bad = kc.batch(kc.A + kc.B, count)
        with pytest.raises(ref.RecordsLimit):
            ref.parse_fetch(srcs[0] + bad, MAX_RECORDS)
        with pytest.raises(EngineError, match="max_records"):
            eng.submit_recordbatch(np.frombuffer(srcs[0] + bad + srcs[1], dtype=np.uint8))
        check(eng, *interleave([("after the refused fetch", srcs[2])], srcs[3:]))
