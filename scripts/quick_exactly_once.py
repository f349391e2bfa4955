"""Cost of exactly-once consumption on a transactional tool Worker (device-template node, three lanes, frame sinks).

Input: `events` tool events dealt over 8 partitions, framed 512 records a frame by the engine's record form (offsets per
partition from 0), landed as one multi-partition fetch per run.  Two legs on the same broker kind
(transactional_id set, so every tick is a transaction in both), alternating, `runs` timed runs each after one warm-up:
  at_least_once    Worker(processing_guarantee="at_least_once"): today's loop
  exactly_once_v2  the same with the consumed positions of every handed-out step sent to the tick's transaction, and the
                   fetch slices kept by the broker until a commit covers them
Per run: the wall time of Worker.run(until_idle=True) (it ends with the lanes drained, i.e. after a device
synchronise) over the ticks it took, and the records per second.  Prints one JSON line with the card name and power
limit read in the same run.

    python scripts/quick_exactly_once.py [events] [runs]
"""
import asyncio
import json
import os
import struct
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "calfkit-sdk_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import tools_def  # noqa: E402
from calfkit import Client, Worker, agent_tool, synth  # noqa: E402
from calfkit.engine import BatchEngine  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 200_000
runs = int(sys.argv[2]) if len(sys.argv) > 2 else 3
IN = "tool.get_weather.input"
FRAME_TOPICS = ["weather_agent.input", "tool.get_weather.output"]
NPARTS, PER_FRAME = 8, 512

recs = synth.tool_events(n, seed=0)
eng = BatchEngine(0, max_records=PER_FRAME, max_in_bytes=16 << 20)
eng.register_topics([IN], num_partitions=0)
buf, parts = b"", []
for p in range(NPARTS):
    parts.append((len(buf), [], p))
    mine, off = recs[p::NPARTS], 0
    for a in range(0, len(mine), PER_FRAME):
        eng.encode_frames_records(IN, [(v, None, None) for v in mine[a:a + PER_FRAME]], 1767225600000)
        fr = eng.fetch_frames()
        for i in range(len(fr)):
            f = fr.frame(i).tobytes()
            buf += struct.pack(">q", off) + f[8:]
            off += struct.unpack_from(">i", f, 57)[0]
        fr.release()
eng.close()


def make(guarantee: str):
    client = Client.connect("localhost", transactional_id=f"bench-{guarantee}")
    sink = {"frames": 0, "bytes": 0}

    def count(topic, part, frame, k):
        sink["frames"] += 1
        sink["bytes"] += int(frame.nbytes)
    for t in FRAME_TOPICS:
        client.broker.frame_sink(t, count)
    node = agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")
    w = Worker(client, nodes=[node], batch_records=1 << 14, batch_bytes=64 << 20, lanes=3,
               route_topics=["weather_agent.input"], processing_guarantee=guarantee)
    return client, w, sink


def one_run(client, w, sink) -> dict:
    client.broker.produce_fetch(IN, buf, partitions=parts)
    steps0, f0 = w.stats["steps"], sink["frames"]
    t0 = time.perf_counter()
    asyncio.run(w.run(until_idle=True))
    dt = time.perf_counter() - t0
    ticks = w.stats["steps"] - steps0
    return {"ms_per_tick": round(dt * 1e3 / ticks, 3), "ticks": ticks, "records_per_s": round(n / dt), "frames": sink["frames"] - f0}


legs = {g: make(g) for g in ("at_least_once", "exactly_once_v2")}
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
res = {"events": n, "fetch_bytes": len(buf), "gpu": q.stdout.strip(), "runs": []}
for g, leg in legs.items():
    one_run(*leg)                                              # warm-up: engines, pinned pools, first launches
t0 = time.time()
for _ in range(runs):
    for g, leg in legs.items():
        res["runs"].append({"leg": g, **one_run(*leg)})
res["wall_s"] = round(time.time() - t0, 1)
committed = legs["exactly_once_v2"][0].broker
group = legs["exactly_once_v2"][1]._subs[0][1].group_id
res["committed_at_end"] = {p: committed.committed(group, IN, p) for p in range(NPARTS)}
print(json.dumps(res))
for _c, w, _s in legs.values():
    w.close()
