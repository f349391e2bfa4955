"""Host side of the LZ4 compression level without a GPU: the broker takes compression_level as it takes
compression_type, the Worker checks it where it checks the codec and hands it to its lane engines and its framer engine,
and a level without compression_type="lz4" changes nothing (Kafka ignores compression.lz4.level for other codecs)."""
import asyncio

import pytest

import calfkit.worker.worker as worker_mod
from calfkit.broker import MemoryBroker
from calfkit.engine.batch import check_compression_level
from calfkit.exceptions import EngineError


def test_memory_broker_and_client_expose_the_level():
    from calfkit import Client
    assert MemoryBroker().compression_level is None
    b = MemoryBroker("localhost", compression_type="lz4", compression_level=9)
    assert b.compression_level == 9 and b.kwargs == {"compression_type": "lz4", "compression_level": 9}
    assert Client.connect("localhost", compression_type="lz4", compression_level=9).broker.compression_level == 9


class _Engine:
    """what the Worker calls on an engine while it configures one; every call is recorded"""
    def __init__(self, *a, **k):
        self.calls, self.topic_ids, self.num_partitions = [], {}, 0
        self.max_payloads = self.max_records = 64
        self.max_in = 1 << 20

    def register_topics(self, topics, num_partitions=0):
        self.topic_ids = {t: i for i, t in enumerate(topics)}
        self.num_partitions = num_partitions

    def encode_frames_records(self, topic, records, ts):
        self.calls.append(("encode_frames_records", topic, len(records)))

    def fetch_frames(self, pool=None):
        return "frames"

    def __getattr__(self, name):
        return lambda *a, **k: self.calls.append((name,) + a)

    def compression(self):
        return [c[1:] for c in self.calls if c[0] == "set_frame_compression"]


class _Pipeline:
    made: list = []

    def __init__(self, device, configure, lanes=1, **kw):
        self.engines = [_Engine() for _ in range(lanes)]
        for e in self.engines:
            configure(e)
        _Pipeline.made.append(self)


def _worker(monkeypatch, frame_sink=True, lanes=2, **kw):
    import tools_def
    from calfkit import Client, Worker, agent_tool
    monkeypatch.setattr(worker_mod, "LanePipeline", _Pipeline)
    monkeypatch.setattr(worker_mod, "BatchEngine", _Engine)
    _Pipeline.made = []
    client = Client.connect("localhost", **kw)
    if frame_sink:
        client.broker.frame_sink("weather_agent.input", lambda *a: None)
    node = agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")
    return Worker(client, nodes=[node], lanes=lanes), node


def _applied(worker, node):
    """(codec, level) each lane engine and the framer engine were given"""
    from calfkit.broker import Record
    worker._pipeline(node)
    lanes = [e.compression() for e in _Pipeline.made[-1].engines]
    assert next(worker._frame_records("weather_agent.input", [Record("weather_agent.input", b"{}")])) == "frames"
    return lanes, worker._framer_eng.compression()


@pytest.mark.parametrize("level", [1, 3, 9, 17])
def test_worker_applies_the_level_to_lane_and_framer_engines(monkeypatch, level):
    worker, node = _worker(monkeypatch, compression_type="lz4", compression_level=level)
    lanes, framer = _applied(worker, node)
    assert lanes == [[("lz4", level)]] * 2 and framer == [("lz4", level)]


def test_worker_without_a_level_keeps_the_default(monkeypatch):
    worker, node = _worker(monkeypatch, compression_type="lz4")
    lanes, framer = _applied(worker, node)
    assert lanes == [[("lz4", None)]] * 2 and framer == [("lz4", None)]


@pytest.mark.parametrize("level", [9, 17])
def test_level_without_lz4_changes_nothing(monkeypatch, level):
    """compression_type=None with a level configures the engines exactly as compression_type=None alone"""
    worker, node = _worker(monkeypatch, compression_level=level)
    with_level = _applied(worker, node)
    worker, node = _worker(monkeypatch)
    assert with_level == _applied(worker, node) == ([[(None, None)]] * 2, [(None, None)])


@pytest.mark.parametrize("level", [0, 18, -1, "9", 9.0, True])
def test_invalid_levels_are_refused_naming_the_value(monkeypatch, level):
    with pytest.raises(EngineError, match=repr(level).replace(".", r"\.")):
        check_compression_level(level)
    worker, _node = _worker(monkeypatch, compression_type="lz4", compression_level=level)
    try:
        with pytest.raises(EngineError, match=repr(level).replace(".", r"\.")):
            asyncio.run(worker.run(until_idle=True))
    finally:
        worker.close()


def test_invalid_level_is_refused_whatever_the_codec(monkeypatch):
    """an out-of-range compression.lz4.level is a configuration error even where it would not apply"""
    worker, _node = _worker(monkeypatch, compression_level=18)
    with pytest.raises(EngineError, match="18"):
        asyncio.run(worker.run(until_idle=True))


def test_no_frame_sinks_no_check(monkeypatch):
    """without frame sinks nothing is framed, so neither the codec nor the level is read"""
    worker, node = _worker(monkeypatch, frame_sink=False, compression_type="lz4", compression_level=18)
    worker._pipeline(node)
    assert _Pipeline.made[-1].engines[0].compression() == []
