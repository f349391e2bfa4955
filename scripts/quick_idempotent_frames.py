"""Cost of idempotent frames on a config-2 step (device-template tool node, 1M events), engine level.

Four legs, alternating, two runs each:
  frames           submit + plan + the frame pass over both output topics + the copy of the frames and their table
  frames_idem      the same with a producer id and epoch in every header (ck_set_producer) and the unkeyed publishes on
                   their topic's sticky partition (ck_set_sticky_partitions, a new one every step), then the host hand-off:
                   every frame's baseSequence written and its CRC32C patched (patch_base_sequence)
  frames_lz4       frames, LZ4-compressed on the device
  frames_lz4_idem  both
Per leg: step time (CUDA events around the whole step, copies included, hand-off excluded), the host hand-off time per
step (a host clock around the patches of all the step's frames), frames per step and frame bytes per step.  Prints one
JSON line with the card name and power limit read in the same run.

    python scripts/quick_idempotent_frames.py [events]
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "calfkit-sdk_b200"))
import torch  # noqa: E402
from calfkit import synth  # noqa: E402
from calfkit.engine import BatchEngine, ToolTemplate  # noqa: E402
from calfkit.engine.batch import patch_base_sequence  # noqa: E402
from calfkit.engine.lane import PinnedPool  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
TOPICS = ["tool.get_weather.input", "tool.get_weather.output", "weather_agent.input"]
FRAME_TOPICS = ["weather_agent.input", "tool.get_weather.output"]
NPARTS = 8
recs = synth.tool_events(n, seed=0)
b = synth.pack(recs)
e = BatchEngine(0, max_records=n, max_in_bytes=b.data.nbytes + 4096)
e.register_topics(TOPICS, num_partitions=NPARTS)
e.set_tool_node("tool.get_weather.output", ToolTemplate.from_format("It's sunny in {location}"))
e.set_frame_topics(FRAME_TOPICS)
d_in, d_off = torch.from_numpy(b.data).cuda(), torch.from_numpy(b.offsets).cuda()
torch.cuda.synchronize()
pool = PinnedPool()
st = torch.cuda.ExternalStream(e.stream_ptr())
seq: dict = {}
sticky_step = [0]


def step(idem: bool):
    e.submit_device(d_in, d_off, n)
    e.tool_plan()
    if idem:
        p = sticky_step[0] % NPARTS
        sticky_step[0] += 1
        e.set_sticky_partitions({t: p for t in FRAME_TOPICS})
    e.encode_frames(1767225600000)
    return e.fetch_frames(pool)


def hand_off(frames) -> None:
    for topic, part, f, k in frames:
        s = seq.get((topic, part), 0)
        patch_base_sequence(f, s)
        seq[(topic, part)] = (s + k) & 0x7FFFFFFF


def leg(name: str, steps: int = 5) -> dict:
    idem = name.endswith("_idem")
    e.set_frame_compression("lz4" if "lz4" in name else None)
    e.set_producer(1000 if idem else -1, 0, False)
    step(idem).release()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms, hand_ms = 0.0, 0.0
    for _ in range(steps):
        ev0.record(st)
        frames = step(idem)
        ev1.record(st)
        torch.cuda.synchronize()
        ms += ev0.elapsed_time(ev1)
        if idem:
            t0 = time.perf_counter()
            hand_off(frames)
            hand_ms += (time.perf_counter() - t0) * 1e3
        nf, fb = len(frames), int(frames.data.nbytes)
        frames.release()
    return {"step_ms": round(ms / steps, 3), "hand_off_ms": round(hand_ms / steps, 3) if idem else None,
            "frames_per_step": nf, "frame_bytes_per_step": fb}


q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
res = {"events": n, "gpu": q.stdout.strip(), "runs": []}
t0 = time.time()
for _ in range(2):
    for name in ("frames", "frames_idem", "frames_lz4", "frames_lz4_idem"):
        res["runs"].append({"leg": name, **leg(name)})
res["wall_s"] = round(time.time() - t0, 1)
print(json.dumps(res))
e.close()
pool.close()
