"""Host side of LZ4 frames without a GPU: the broker takes compression_type as a FastStream KafkaBroker does, and a Worker
with frame sinks refuses, when it builds a pipeline, any codec the device does not build."""
import asyncio

import pytest

from calfkit.broker import MemoryBroker
from calfkit.exceptions import EngineError


def test_memory_broker_exposes_the_codec():
    from calfkit import Client
    assert MemoryBroker().compression_type is None
    b = MemoryBroker("localhost", compression_type="lz4")
    assert b.compression_type == "lz4" and b.kwargs == {"compression_type": "lz4"}
    assert Client.connect("localhost", compression_type="lz4").broker.compression_type == "lz4"


def _worker(codec, frame_sink=True):
    import tools_def
    from calfkit import Client, Worker, agent_tool
    client = Client.connect("localhost", compression_type=codec)
    if frame_sink:
        client.broker.frame_sink("weather_agent.input", lambda *a: None)
    return Worker(client, nodes=[agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")])


@pytest.mark.parametrize("codec", ["zstd", "gzip", "snappy", "LZ4", "none"])
def test_worker_refuses_codecs_the_device_does_not_build(codec):
    worker = _worker(codec)
    try:
        with pytest.raises(EngineError, match=codec):
            asyncio.run(worker.run(until_idle=True))
    finally:
        worker.close()


@pytest.mark.parametrize("codec", [None, "lz4"])
def test_worker_frame_codec_is_the_brokers(codec):
    worker = _worker(codec)
    try:
        assert worker._frame_codec() == codec
    finally:
        worker.close()
