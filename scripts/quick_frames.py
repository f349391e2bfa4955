"""Cost of the frame pass on a config-2 step (device-template tool node, 1M events), engine level.

Five legs, alternating, two runs each:
  sink           submit + plan + the copies a producer reads today (payload arena, offsets, lengths, publish table)
  frames         the same + the frame pass over both output topics + the copy of the frames and their table
  frames_lz4     the same with LZ4 frames (ck_set_option 3 = 3): the frames are compressed on the device before the copy
  frames_lz4_l3  the same at compression level 3 (ck_set_option 4: the hash-chain parse, 4 candidates per position)
  frames_lz4_l9  the same at compression level 9 (256 candidates per position, the deepest search)
Per leg: step time (CUDA events around the whole step, copies included), the frame pass's kernel time (profile timer
"frame") and the compressor's ("lz4"), events/s, frame bytes and D2H bytes per step, and the compression ratio
(uncompressed / compressed frame bytes) of each LZ4 leg.  Where liblz4 is installed, the sizes of liblz4's LZ4F frames at
levels 1, 3 and 9 over the same records sections (64 KB independent blocks; a comparison only).  Prints one JSON line with
the card name and power limit read in the same run.

    python scripts/quick_frames.py [events]
"""
import ctypes as C
import ctypes.util
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


LEGS = {"sink": (None, None), "frames": (None, None), "frames_lz4": ("lz4", None), "frames_lz4_l3": ("lz4", 3), "frames_lz4_l9": ("lz4", 9)}


def leg(name: str, steps: int = 5) -> dict:
    frames = name != "sink"
    e.set_frame_compression(*LEGS[name])
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
    for name in LEGS:
        res["runs"].append({"leg": name, **leg(name)})
res["wall_s"] = round(time.time() - t0, 1)
size = {name: next(r["frame_bytes_per_step"] for r in res["runs"] if r["leg"] == name) for name in LEGS}
res["frames_per_step"] = e.frames_size()[0]
res["compression_ratio"] = {name: round(size["frames"] / size[name], 2) for name in LEGS if name.startswith("frames_lz4")}
res["size_vs_greedy"] = {name: round(size[name] / size["frames_lz4"], 4) for name in ("frames_lz4_l3", "frames_lz4_l9")}


def liblz4_sizes(levels) -> dict | None:
    """bytes of the frames with each records section as one LZ4F frame of liblz4 at each level (64 KB independent blocks,
    no checksums: the device's frame format), over the frames of one uncompressed pass of the same step"""
    name = ctypes.util.find_library("lz4")
    if not name:
        return None
    L = C.CDLL(name)
    L.LZ4F_compressFrameBound.restype = C.c_size_t
    L.LZ4F_compressFrameBound.argtypes = [C.c_size_t, C.c_void_p]
    L.LZ4F_compressFrame.restype = C.c_size_t
    L.LZ4F_compressFrame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.LZ4F_isError.argtypes = [C.c_size_t]
    e.set_frame_compression(None)
    step(True)
    fr = e.fetch_frames()
    sections = [f[61:].tobytes() for _t, _p, f, _n in fr]
    fr.release()
    from concurrent.futures import ThreadPoolExecutor
    out = {}
    for level in levels:
        prefs = (C.c_int * 14)()                          # LZ4F_preferences_t: frameInfo (32 bytes), level, autoFlush, ...
        prefs[0], prefs[1], prefs[8] = 4, 1, level        # blockSizeID 4 (64 KB), blockMode 1 (independent), compressionLevel

        def one(sec, prefs=prefs):
            cap = L.LZ4F_compressFrameBound(len(sec), prefs)
            dst = C.create_string_buffer(cap)
            r = L.LZ4F_compressFrame(dst, cap, sec, len(sec), prefs)
            assert not L.LZ4F_isError(r)
            return 61 + r
        with ThreadPoolExecutor(os.cpu_count()) as pool:
            out[f"level_{level}"] = sum(pool.map(one, sections))
    return out


res["liblz4_frame_bytes"] = liblz4_sizes((1, 3, 9))
print(json.dumps(res))
