"""Cost of the frame pass on a config-2 step (device-template tool node, 1M events), engine level.

Three legs, alternating, two runs each:
  sink        submit + plan + the copies a producer reads today (payload arena, offsets, lengths, publish table)
  frames      the same + the frame pass over both output topics + the copy of the frames and their table
  frames_lz4  the same with LZ4 frames (ck_set_option 3 = 3): the frames are compressed on the device before the copy
Per leg: step time (CUDA events around the whole step, copies included), the frame pass's kernel time (profile timer
"frame") and the compressor's ("lz4"), events/s, frame bytes and D2H bytes per step, and the compression ratio
(uncompressed / compressed frame bytes).  Prints one JSON line with the card name and power limit read in the same run.

    python scripts/quick_frames.py [events]
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "calfkit-sdk_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from calfkit import synth  # noqa: E402
from calfkit.engine import BatchEngine, ToolTemplate  # noqa: E402
from calfkit.engine._lib import FRAME_DTYPE, PUB_DTYPE, ptr  # noqa: E402
from calfkit.engine.lane import PinnedBuffer  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
recs = synth.tool_events(n, seed=0)
b = synth.pack(recs)
e = BatchEngine(0, max_records=n, max_in_bytes=b.data.nbytes + 4096)
e.register_topics(["tool.get_weather.input", "tool.get_weather.output", "weather_agent.input"], num_partitions=8)
e.set_tool_node("tool.get_weather.output", ToolTemplate.from_format("It's sunny in {location}"))
e.set_frame_topics(["weather_agent.input", "tool.get_weather.output"])
d_in, d_off = torch.from_numpy(b.data).cuda(), torch.from_numpy(b.offsets).cuda()
torch.cuda.synchronize()
b_out = PinnedBuffer(e.max_out + 64)
b_off, b_len = PinnedBuffer(8 * (n + 1)), PinnedBuffer(4 * n)
b_pubs = PinnedBuffer(PUB_DTYPE.itemsize * 2 * n)
b_fr, b_tab = PinnedBuffer(2 * e.max_out + 160 * 2 * n), PinnedBuffer(FRAME_DTYPE.itemsize * 2 * n)
st = torch.cuda.ExternalStream(e.stream_ptr())


def step(frames: bool) -> tuple[int, int]:
    e.submit_device(d_in, d_off, n)
    e.tool_plan()
    if frames:
        e.encode_frames(1767225600000)
    nb, npay, npub = e.out_size()
    e._check(e.lib.ck_fetch_output_async(e.h, ptr(b_out.array), b_out.nbytes, ptr(b_off.array), ptr(b_len.array), ptr(b_pubs.array)))
    d2h, fb = nb + 8 * (npay + 1) + 4 * npay + PUB_DTYPE.itemsize * npub, 0
    if frames:
        nf, fb = e.frames_size()
        e._check(e.lib.ck_fetch_frames_async(e.h, ptr(b_tab.array), 2 * n, ptr(b_fr.array), b_fr.nbytes))
        d2h += fb + FRAME_DTYPE.itemsize * nf
    e.sync()
    return d2h, fb


def leg(name: str, steps: int = 5) -> dict:
    frames = name != "sink"
    e.set_frame_compression("lz4" if name == "frames_lz4" else None)
    step(frames)
    e.profile(True)
    e.profile_read()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(st)
    for _ in range(steps):
        d2h, fb = step(frames)
    ev1.record(st)
    torch.cuda.synchronize()
    prof = e.profile_read()
    e.profile(False)
    ms = ev0.elapsed_time(ev1) / steps
    return {"step_ms": round(ms, 3), "frame_kernel_ms": round(prof["frame"][0] / steps, 3),
            "lz4_kernel_ms": round(prof["lz4"][0] / steps, 3), "events_per_s": round(n / ms * 1e3),
            "frame_bytes_per_step": fb, "d2h_bytes_per_step": d2h}


q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
res = {"events": n, "gpu": q.stdout.strip(), "runs": []}
t0 = time.time()
for _ in range(2):
    for name in ("sink", "frames", "frames_lz4"):
        res["runs"].append({"leg": name, **leg(name)})
res["wall_s"] = round(time.time() - t0, 1)
raw = next(r["frame_bytes_per_step"] for r in res["runs"] if r["leg"] == "frames")
comp = next(r["frame_bytes_per_step"] for r in res["runs"] if r["leg"] == "frames_lz4")
res["frames_per_step"] = e.frames_size()[0]
res["compression_ratio"] = round(raw / comp, 2)
print(json.dumps(res))
