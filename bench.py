#!/usr/bin/env python
"""bench.py — agent-events/sec of the calfkit hot path on H100 (BASELINE.json metric).

    python bench.py --gpus 1 --steps 10 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N --steps K --warmup W
    python bench.py --impl reference ...        # the reference's CPU path (oracle port) on the host cores
    python bench.py ... --dump-outputs DIR      # + the last timed step's outputs as DIR/<name>.npy (seeded inputs)

One "step" = one pass of the tool-node hot path (decode -> ToolNodeDef.run -> _publish_action ->
encode -> route) over one batch of `--events` synthetic 1 KB-class agent events per GPU
(BASELINE.json configs[1]: "1M synthetic 1 KB agent-event JSON, single @agent_tool node").
`value`     : whole-job events/s with the batch resident in HBM when the timed region starts.
`e2e`       : the same through the public BatchEngine API with pinned HOST buffers — H2D of the
              batch and D2H of every payload + the publish table inside the timed region.
`roofline`  : dominant kernel, algorithmic bytes / its CUDA-event duration (events recorded on the
              engine's own stream inside the timed region) vs the HBM peak (MEASURED_PEAKS.json, else the data sheet).
`cpu_baseline`: the oracle port (reference algorithm on pydantic-core) on all host cores, bounded sample.
N > 1: records shard by Kafka partition (murmur2(correlation_id) % 8 -> GPU), weak scaling; a
fraction (--cross, default 1/8) of each rank's records arrive on the "wrong" partition (the
reference's unkeyed first publish, client/base.py:147) and their keyed outputs are forwarded to the
owning GPU with one variable-size NCCL all-to-all per step.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "calfkit-sdk_b200"))
sys.path.insert(0, ROOT)

METRIC = "agent_events_per_sec"
UNIT = "events/s"
NUM_PARTITIONS = 8
TOOL_FMT = "It's sunny in {location}"


# ------------------------------------------------------------------------------------------------ CPU arm
def _cpu_worker(chunk):
    from oracle import port
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import tools_def
    node = port.ToolNode.of(tools_def.get_weather)
    nbytes = 0
    for rec in chunk:
        for (_t, _k, _c, payload) in port.tool_node_event(node, rec):
            nbytes += len(payload)
    return len(chunk), nbytes


def cpu_arm(records, cores: int, start: str = "fork"):
    """events/s of the oracle port over `records`, split over `cores` processes."""
    import multiprocessing as mp
    chunks = [records[i::cores] for i in range(cores)]
    ctx = mp.get_context(start)
    with ctx.Pool(cores) as pool:
        pool.map(_cpu_worker, [c[:8] for c in chunks])          # import + warm-up outside the timing
        t0 = time.perf_counter()
        res = pool.map(_cpu_worker, chunks)
        dt = time.perf_counter() - t0
    n = sum(r[0] for r in res)
    return n / dt, dt, n


class ReferencePool:
    """worker processes running the UNMODIFIED reference (oracle/_ref mirror, or /root/reference in the build
    container); the oracle port when no reference tree is present.  kind = "reference" | "port"."""
    def __init__(self, cores: int):
        from oracle import ref_harness, ref_runner
        self.kind = "reference" if ref_harness.available() else "port"
        self.pool = ref_runner.Pool(cores, None if self.kind == "reference" else _cpu_worker)
        self.cores = cores

    def run(self, records):
        return self.pool.run(records)

    def close(self):
        self.pool.close()

    def describe(self) -> str:
        return ("unmodified reference code (oracle/_ref mirror of /root/reference/calfkit): Envelope.model_validate_json -> "
                "ToolNodeDef.handler -> _publish_action -> model_dump_json, sync tool on the anyio thread as in the stock path"
                if self.kind == "reference" else "oracle/port.py (no reference tree present)")


WORKLOADS = {
    "tool_event_1k": "tool_event_1k: tool-stage Envelope JSON (1152+-16 B), single @agent_tool node get_weather (BASELINE.json configs[1])",
    "fanout": "fanout: 1 Agent node -> F @agent_tool nodes (BASELINE.json configs[2]), post-LLM agent-stage envelopes",
    "reply": "reply: client-side projection of final reply envelopes to NodeResult.output (SURVEY 8f row 3)",
    "mixed": "mixed: sizes log-uniform 128 B-64 KB, 256 subscribe_topics (BASELINE.json configs[4])",
}


def bench_config(args, world: int) -> dict:
    """the `config` object of the JSON line: a pure function of the command line, identical on both arms"""
    return {"workload": WORKLOADS[args.workload], "events_per_gpu_per_step": args.events, "seed": 1000,
            "partitions": NUM_PARTITIONS, "cross_partition_fraction": args.cross if world > 1 else 0.0,
            "sharding": "records by Kafka partition -> GPU" if world > 1 else "single GPU",
            "tool": "device template " + repr(TOOL_FMT),
            "l2": "inputs and outputs per step (> 1 GB each at 1 M events) far exceed the 50 MB L2: every step streams from HBM",
            "broker_io": "excluded on both arms (FastStream/aiokafka are not installable offline)"}


def run_reference(args, rank: int, world: int) -> None:
    """the reference's own CPU implementation of the path (oracle/ref_runner.py: validate -> ToolNodeDef.handler ->
    _publish_action -> dump, unmodified reference code) on all host cores; each step a bounded sample of the SAME
    seeded batch the GPU arm consumes"""
    if rank != 0:
        return
    from calfkit import synth
    cores = os.cpu_count() or 1
    per_step = min(args.events, max(cores * 400, 4000))           # ~1-2 s of work per step on all cores
    recs = synth.tool_events(per_step, seed=1000)                  # = the first per_step records of the GPU arm's rank-0 batch
    pool = ReferencePool(cores)
    for _ in range(max(args.warmup, 1)):
        pool.run(recs[: max(cores * 8, 64)])
    t_total, n_total, kind = 0.0, 0, pool.kind
    for _ in range(args.steps):
        _v, dt, n = pool.run(recs)
        t_total += dt
        n_total += n
    pool.close()
    value = n_total / t_total
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": 1e3 * t_total / args.steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": bench_config(args, world),
        "cpu_baseline": {"value": value, "unit": UNIT, "cores": cores, "kind": kind,
                         "sample": f"first {per_step} events of the batch per step x {args.steps} steps over {cores} processes; "
                                   + pool.describe()},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


def hbm_peak_gbs():
    """-> (GB/s, where it came from): the driver-written measurement if present and sane, else the data-sheet figure"""
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        v = float(json.load(open(path))["hbm_gbs"])
        if v > 0:
            return v, "measured (MEASURED_PEAKS.json hbm_gbs, burst copy)"
    except Exception:  # noqa: BLE001  (absent / unreadable / other schema)
        pass
    return 3350.0, "data sheet (H100 SXM HBM3, 3.35 TB/s at 700 W; not measured)"


# ------------------------------------------------------------------------------------------------ helpers
def teardown(world: int) -> None:
    import torch
    torch.cuda.synchronize()
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


class ClockSampler(threading.Thread):
    def __init__(self, index: int):
        super().__init__(daemon=True)
        self.index, self.samples, self.reasons, self.stop_flag, self.max_mhz = index, [], set(), False, None
        self.gpu = self.power_limit_w = None
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.dev = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self.dev, pynvml.NVML_CLOCK_SM)
            self.gpu = pynvml.nvmlDeviceGetName(self.dev)
            self.gpu = self.gpu.decode() if isinstance(self.gpu, bytes) else self.gpu
            self.power_limit_w = pynvml.nvmlDeviceGetEnforcedPowerLimit(self.dev) / 1000
        except Exception:
            self.nv = None

    def run(self):
        if self.nv is None:
            return
        nv = self.nv
        names = {"hw_slowdown": 0x8, "sw_power_cap": 0x4, "hw_thermal_slowdown": 0x40, "sw_thermal_slowdown": 0x20,
                 "hw_power_brake_slowdown": 0x80, "sync_boost": 0x10, "applications_clocks_setting": 0x2}
        while not self.stop_flag:
            try:
                self.samples.append(nv.nvmlDeviceGetClockInfo(self.dev, nv.NVML_CLOCK_SM))
                try:
                    r = nv.nvmlDeviceGetCurrentClocksEventReasons(self.dev)
                except Exception:
                    r = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.dev)
                for k, bit in names.items():
                    if r & bit:
                        self.reasons.add(k)
            except Exception:
                pass
            time.sleep(0.004)

    def summary(self):
        s = sorted(self.samples)
        return {"gpu": self.gpu, "power_limit_w": self.power_limit_w, "sm_mhz": s[len(s) // 2] if s else None,
                "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons), "samples": len(s)}


def dump_outputs(eng, path: str) -> None:
    """--dump-outputs: what the engine's last plan produced, as float .npy files under 64 MB in all, so that two builds
    can be compared output for output: length and CRC-32 of every payload, the first 1 KB of a seeded sample of payloads
    (chosen by index only; -1 pads), the publish table and per-record status / action.  A table longer than its cap is a
    seeded sample of rows, listed in <name>_index.npy."""
    import zlib
    import numpy as np
    from calfkit.engine._lib import COL
    out, off, ln, pubs = eng._fetch()
    cols = eng.columns()
    rng = np.random.default_rng(0)
    arrays = {}

    def rows(name: str, m: int, cap: int) -> np.ndarray:
        if m <= cap:
            return np.arange(m)
        idx = np.sort(rng.choice(m, size=cap, replace=False))
        arrays[name + "_index"] = idx.astype(np.float64)
        return idx

    mv = memoryview(out)
    pr = rows("payload", len(ln), 1 << 20)
    arrays["payload_len"] = ln[pr].astype(np.float32)
    arrays["payload_crc32"] = np.array([zlib.crc32(mv[off[i]:off[i] + ln[i]]) for i in pr], dtype=np.float64)
    take = np.sort(rng.choice(len(ln), size=min(len(ln), 4096), replace=False))
    head = np.full((len(take), 1024), -1.0, dtype=np.float32)
    for j, i in enumerate(take):
        k = min(int(ln[i]), 1024)
        head[j, :k] = out[off[i]:off[i] + k]
    arrays["payload_sample_index"], arrays["payload_sample_head"] = take.astype(np.float64), head
    fields = ("payload", "topic_id", "topic_off", "topic_len", "record", "has_key", "partition")
    pi = rows("publishes", len(pubs), 1 << 17)
    arrays["publishes"] = np.stack([pubs[f][pi].astype(np.float64) for f in fields], axis=1) if len(pi) \
        else np.zeros((0, len(fields)), np.float64)
    ri = rows("record", cols.shape[1], 1 << 20)
    arrays["record_status"], arrays["record_action"] = (cols[COL[c]][ri].astype(np.float32) for c in ("STATUS", "ACTION"))
    total = sum(a.nbytes for a in arrays.values())
    assert total <= 64 << 20, total
    os.makedirs(path, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(path, name + ".npy"), a)


class CudaArray:
    """wraps a raw device pointer for torch.as_tensor via __cuda_array_interface__"""
    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = {"data": (ptr, False), "shape": tuple(shape), "typestr": typestr, "version": 3}


def np_murmur2_32(keys):
    """vectorised Kafka murmur2 over fixed-width keys: uint8 [n, L] with L % 4 == 0"""
    import numpy as np
    n, L = keys.shape
    w = keys.reshape(n, L // 4, 4).astype(np.uint32)
    k = w[:, :, 0] | (w[:, :, 1] << 8) | (w[:, :, 2] << 16) | (w[:, :, 3] << 24)
    m = np.uint32(0x5BD1E995)
    h = np.full(n, np.uint32(0x9747B28C) ^ np.uint32(L), dtype=np.uint32)
    with np.errstate(over="ignore"):
        for i in range(L // 4):
            kk = k[:, i] * m
            kk ^= kk >> np.uint32(24)
            kk *= m
            h *= m
            h ^= kk
        h ^= h >> np.uint32(13)
        h *= m
        h ^= h >> np.uint32(15)
    return h


def place_on_partitions(batch, corr_off, rank: int, world: int, cross: float, seed: int):
    """Rewrites each record's 32-hex correlation id in place so that murmur2(id) % 8 % world == rank
    for (1 - cross) of the records and != rank for the rest (arrived on the 'wrong' partition)."""
    import numpy as np
    rng = np.random.default_rng(seed)
    n = batch.n
    data = batch.data.copy()
    want_home = np.full(n, rank, dtype=np.int64)
    if world > 1:
        away = rng.random(n) < cross
        want_home[away] = (rank + 1 + rng.integers(0, world - 1, size=int(away.sum()))) % world
    pos = batch.offsets[:-1] + corr_off.astype(np.int64)
    todo = np.arange(n)
    hexd = np.frombuffer(b"0123456789abcdef", dtype=np.uint8)
    while todo.size:
        cand = hexd[rng.integers(0, 16, size=(todo.size, 32))]
        home = (np_murmur2_32(cand) & np.uint32(0x7FFFFFFF)) % np.uint32(NUM_PARTITIONS) % np.uint32(world)
        ok = home == want_home[todo]
        idx = todo[ok]
        if idx.size:
            cols = pos[idx][:, None] + np.arange(32)[None, :]
            data[cols] = cand[ok]
        todo = todo[~ok]
    batch.data = data
    return batch



def _cpu_fanout_worker(chunk):
    from oracle import port
    registry = {f"tool_{j:02d}": f"tool.tool_{j:02d}.input" for j in range(256)}
    nb = 0
    for rec in chunk:
        for (_t, _k, _c, payload) in port.agent_fanout("planner", "planner.input", "planner.output", registry, rec):
            nb += len(payload)
    return len(chunk), nb


def run_fanout(args, rank, world, local_rank, dev, real_stdout, all_cpus=None) -> None:
    """BASELINE.json configs[2]: one Agent node fans every event out to F @agent_tool nodes (reference
    nodes/agent.py:177-211 + nodes/base.py:73-88): per event F envelopes, each the full state + one pushed frame,
    plus the handler-return publish of the original envelope.  Write-bandwidth bound."""
    import multiprocessing as mp
    import numpy as np
    import torch
    from calfkit import synth
    from calfkit.engine import BatchEngine
    F = args.fanout
    n = args.events if args.events != 1_000_000 else 4096
    recs = synth.fanout_events(n, seed=3000 + rank, fanout=F)
    batch = synth.pack(recs)
    in_bytes = int(batch.data.nbytes)
    per_out = int(in_bytes / n) + 260
    out_cap = n * ((F + 1) * (per_out + 16)) + (1 << 20)
    eng = BatchEngine(local_rank, max_records=n, max_in_bytes=in_bytes + 4096, max_out_bytes=out_cap, max_payloads=n * (F + 1))
    registry = {f"tool_{j:02d}": f"tool.tool_{j:02d}.input" for j in range(F)}
    eng.register_topics(list(registry.values()) + ["planner.input", "planner.output"], num_partitions=NUM_PARTITIONS)
    eng.set_agent_node("planner", "planner.input", "planner.output", registry)
    d_in = torch.from_numpy(batch.data.copy()).to(dev)
    d_off = torch.from_numpy(batch.offsets.copy()).to(dev)
    stream = torch.cuda.ExternalStream(eng.stream_ptr(), device=dev)
    ms0 = 1767225600000

    def step(k):
        eng.submit_device(d_in, d_off, n)
        eng.fanout_plan(ms0 + k, 1234 + k, max_fanout=256)

    for k in range(args.warmup):
        step(k)
    eng.sync()
    eng.profile(True)
    sampler = ClockSampler(local_rank)
    sampler.start()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    l0 = eng.launch_count()
    ev0.record(stream)
    for k in range(args.steps):
        step(k)
    ev1.record(stream)
    torch.cuda.synchronize()
    sampler.stop_flag = True
    gpu_launches = eng.launch_count() - l0
    ms_step = ev0.elapsed_time(ev1) / args.steps
    prof = eng.profile_read()
    eng.profile(False)
    out_bytes, npay, npub = eng.out_size()
    value = world * n / (ms_step / 1e3)
    if args.dump_outputs and rank == 0:
        dump_outputs(eng, args.dump_outputs)
    # end to end: pinned host in -> device -> pinned host out
    h_in = torch.from_numpy(batch.data.copy()).pin_memory()
    h_off = torch.from_numpy(batch.offsets.copy()).pin_memory()
    h_out = torch.empty(out_bytes + (1 << 20), dtype=torch.uint8).pin_memory()
    h_o = torch.empty(npay + 1, dtype=torch.int64).pin_memory().numpy()
    h_l = torch.empty(npay, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    from calfkit.engine._lib import PUB_DTYPE
    h_p = torch.empty(npub * PUB_DTYPE.itemsize, dtype=torch.uint8).pin_memory().numpy().view(PUB_DTYPE)
    d2h = 0
    for k in range(2):
        eng.submit(h_in.numpy(), h_off.numpy()); eng.fanout_plan(ms0, 1, max_fanout=256)
        o, of, ln, pb = eng._fetch(out_buf=h_out.numpy(), off_buf=h_o, len_buf=h_l, pubs_buf=h_p)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e2e_steps = args.steps
    for k in range(e2e_steps):
        eng.submit(h_in.numpy(), h_off.numpy()); eng.fanout_plan(ms0, 1, max_fanout=256)
        o, of, ln, pb = eng._fetch(out_buf=h_out.numpy(), off_buf=h_o, len_buf=h_l, pubs_buf=h_p)
        d2h = int(o.nbytes + of.nbytes + ln.nbytes + pb.nbytes)
    torch.cuda.synchronize()
    e2e_ms = (time.perf_counter() - t0) * 1e3 / e2e_steps
    payload_bytes = int(ln.astype(np.int64).sum())
    peak, _peak_src = hbm_peak_gbs()
    kern = {k: {"ms_per_launch": ms / c, "launches": c} for k, (ms, c) in prof.items() if c}
    emit_ms = kern["emit"]["ms_per_launch"]
    algo_emit = in_bytes + payload_bytes            # every input byte read at least once + every payload byte written
    # parity spot check (byte-exact, outside the timed regions): the first events' F Call envelopes + handler return vs the oracle
    from oracle import port
    from calfkit import _ids
    from calfkit.engine.batch import device_uuid7_hex
    small = synth.pack(recs[:4])
    eng.submit(small.data, small.offsets)
    eng.fanout_plan(ms0, 99, max_fanout=256)
    chk = list(eng.fetch().publishes())
    parity_ok, kk, slot = True, 0, 0
    for rec in recs[:4]:
        it = iter([device_uuid7_hex(ms0, 99, slot + j) for j in range(F)])
        _ids.set_id_source(lambda: next(it))
        try:
            want = port.agent_fanout("planner", "planner.input", "planner.output", registry, rec)
        finally:
            _ids.set_id_source(None)
        parity_ok = parity_ok and [(p.topic, p.key, p.payload) for p in chk[kk:kk + len(want)]] == [(t, k2, pl) for (t, k2, _c, pl) in want]
        kk += len(want)
        slot += F + 1
    cores = os.cpu_count() or 1
    sample = recs[: max(cores * 2, 64)]
    if all_cpus:
        os.sched_setaffinity(0, all_cpus)
    ctx = mp.get_context("spawn")
    with ctx.Pool(min(cores, len(sample))) as pool:
        chunks = [sample[i::cores] for i in range(cores) if sample[i::cores]]
        pool.map(_cpu_fanout_worker, [c[:1] for c in chunks])
        t0 = time.perf_counter()
        res = pool.map(_cpu_fanout_worker, chunks)
        cpu_dt = time.perf_counter() - t0
    cpu_n = sum(r[0] for r in res)
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_step,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": dict(bench_config(args, world), fanout=F, events_per_gpu_per_step=n),
        "workload_stats": {"record_bytes_mean": in_bytes / n, "payloads_per_event": npay / n, "out_bytes_per_event": payload_bytes / n,
                           "out_gb_per_step": payload_bytes / 1e9, "parity_spot_check_4_events": parity_ok},
        "clocks": sampler.summary(),
        "e2e": {"value": world * n / (e2e_ms / 1e3), "unit": UNIT, "h2d_bytes_per_step": in_bytes + 8 * (n + 1), "d2h_bytes_per_step": d2h,
                "ms_per_step": e2e_ms, "steps": e2e_steps, "api": "BatchEngine.submit(pinned host) + fanout_plan + fetch(pinned host)"},
        "gpu_launches": gpu_launches,
        "roofline": {"kernel": "ck_emit_kernel", "bound": "hbm", "achieved": algo_emit / emit_ms / 1e6, "peak": peak, "unit": "GB/s",
                     "frac": algo_emit / emit_ms / 1e6 / peak, "traffic": None, "share_of_step": emit_ms / ms_step, "kernels": kern,
                     "dominant_by_time": max(kern, key=lambda k_: kern[k_]["ms_per_launch"] * (2 if k_ == "fanout" else 1)),
                     "pipeline": {"algo_bytes_per_event": (in_bytes + payload_bytes) / n, "achieved": (in_bytes + payload_bytes) / ms_step / 1e6,
                                  "frac": (in_bytes + payload_bytes) / ms_step / 1e6 / peak}},
        "cpu_baseline": {"value": cpu_n / cpu_dt, "unit": UNIT, "cores": cores, "kind": "port",
                         "sample": f"{cpu_n} events in {cpu_dt:.1f} s over {min(cores, len(sample))} processes (oracle/port.py agent_fanout)"},
    }
    sys.stdout.flush()
    os.write(real_stdout, (json.dumps(line) + "\n").encode())
    torch.cuda.synchronize()
    del stream
    eng.close()
    teardown(world)


def _cpu_reply_worker(chunk):
    from oracle import port
    n = 0
    for r in chunk:
        try:
            port.reply_output(r)
        except Exception:  # noqa: BLE001  (DeserializationError is part of the path)
            pass
        n += 1
    return n, 0


def run_reply(args, rank, world, local_rank, dev, real_stdout, all_cpus=None) -> None:
    """SURVEY.md section 8f row 3, the client reply path (reference client/deserialize.py:15-89): every step validates a
    batch of final reply envelopes and extracts NodeResult.output (first DataPart.data, else first TextPart.text)."""
    import multiprocessing as mp
    import random
    import numpy as np
    import torch
    from calfkit import synth
    from calfkit.engine import BatchEngine
    n = args.events
    rng = random.Random(7 + rank)
    base = synth.tool_events(min(n, 20000), seed=4000 + rank)
    recs = []
    for i in range(n):
        r = base[i % len(base)]
        k = rng.randrange(4)
        parts = [] if k == 0 else ['{"kind":"text","text":"It\'s sunny in %s","metadata":null}' % ("x" * rng.randrange(4, 40))]
        if k >= 2:
            parts.insert(rng.randrange(2), '{"kind":"data","data":{"temp":%d,"ok":true,"tags":["a","b"]},"schema_":null,"metadata":null}' % rng.randrange(40))
        recs.append(r.replace(b'"final_output_parts":[]', ('"final_output_parts":[' + ",".join(parts) + "]").encode()))
    batch = synth.pack(recs)
    in_bytes = int(batch.data.nbytes)
    eng = BatchEngine(local_rank, max_records=n, max_in_bytes=in_bytes + 4096, max_out_bytes=n * 272 + (1 << 20))
    eng.set_bucketing(True)            # four reply shapes mixed in every warp: bucket by length before the walk
    d_in = torch.from_numpy(batch.data.copy()).to(dev)
    d_off = torch.from_numpy(batch.offsets.copy()).to(dev)
    stream = torch.cuda.ExternalStream(eng.stream_ptr(), device=dev)

    def step():
        eng.submit_device(d_in, d_off, n)
        eng.reply_plan(0)

    for _ in range(args.warmup):
        step()
    eng.sync()
    eng.profile(True)
    sampler = ClockSampler(local_rank)
    sampler.start()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    l0 = eng.launch_count()
    ev0.record(stream)
    for _ in range(args.steps):
        step()
    ev1.record(stream)
    torch.cuda.synchronize()
    sampler.stop_flag = True
    gpu_launches = eng.launch_count() - l0
    ms_step = ev0.elapsed_time(ev1) / args.steps
    prof = eng.profile_read()
    eng.profile(False)
    out_bytes, npay, _npub = eng.out_size()
    value = world * n / (ms_step / 1e3)
    if args.dump_outputs and rank == 0:
        dump_outputs(eng, args.dump_outputs)
    h_in = torch.from_numpy(batch.data.copy()).pin_memory()
    h_off = torch.from_numpy(batch.offsets.copy()).pin_memory()
    h_out = torch.empty(out_bytes + (1 << 20), dtype=torch.uint8).pin_memory()
    h_o = torch.empty(npay + 1, dtype=torch.int64).pin_memory().numpy()
    h_l = torch.empty(npay, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    d2h = 0
    e2e_steps = args.steps
    for k in range(2 + e2e_steps):
        if k == 2:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        eng.submit(h_in.numpy(), h_off.numpy()); eng.reply_plan(0)
        o, of, ln, pb = eng._fetch(out_buf=h_out.numpy(), off_buf=h_o, len_buf=h_l)
        d2h = int(o.nbytes + of.nbytes + ln.nbytes)
    torch.cuda.synchronize()
    e2e_ms = (time.perf_counter() - t0) * 1e3 / e2e_steps
    cols = eng.columns()
    peak, _peak_src = hbm_peak_gbs()
    kern = {k: {"ms_per_launch": ms / c, "launches": c, "ms_per_step": ms / args.steps} for k, (ms, c) in prof.items() if c}
    walk_ms = kern["walk"]["ms_per_step"]              # bucketing is on: the two sort passes are timed with the walk they serve
    from calfkit.engine._lib import COL as _COL, NUM_COLS as _NC
    algo_walk = in_bytes + 8 * (n + 1) + 4 * (_NC - 10) * n            # the walker writes every column but the plan kernels'
    # parity spot check against the oracle (byte-exact), outside the timed regions
    from oracle import port
    small = synth.pack(recs[:256])
    eng.submit(small.data, small.offsets); eng.reply_plan(0)
    chk = eng.fetch()
    ok = True
    for i, r in enumerate(recs[:256]):
        try:
            want = port.reply_output(r)[1]
        except Exception:  # noqa: BLE001
            want = b""
        ok = ok and chk.payload(i) == want
    cores = os.cpu_count() or 1
    sample = recs[: max(cores * 400, 4000)]
    if all_cpus:
        os.sched_setaffinity(0, all_cpus)
    ctx = mp.get_context("spawn")
    with ctx.Pool(cores) as pool:
        chunks = [sample[i::cores] for i in range(cores) if sample[i::cores]]
        pool.map(_cpu_reply_worker, [c[:2] for c in chunks])
        t0 = time.perf_counter()
        res = pool.map(_cpu_reply_worker, chunks)
        cpu_dt = time.perf_counter() - t0
    cpu_n = sum(r[0] for r in res)
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_step,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": bench_config(args, world),
        "workload_stats": {"record_bytes_mean": in_bytes / n, "out_bytes_per_event": out_bytes / n,
                           "ok_fraction": float((cols[_COL["STATUS"]] == 0).mean()), "parity_vs_oracle_256": ok, "in_gb_per_step": in_bytes / 1e9},
        "clocks": sampler.summary(),
        "e2e": {"value": world * n / (e2e_ms / 1e3), "unit": UNIT, "h2d_bytes_per_step": in_bytes + 8 * (n + 1), "d2h_bytes_per_step": d2h,
                "ms_per_step": e2e_ms, "steps": e2e_steps, "api": "BatchEngine.submit(pinned host) + reply_plan + fetch(pinned host)"},
        "gpu_launches": gpu_launches,
        "roofline": {"kernel": "ck_walk_kernel", "bound": "hbm", "achieved": algo_walk / walk_ms / 1e6, "peak": peak, "unit": "GB/s",
                     "frac": algo_walk / walk_ms / 1e6 / peak, "traffic": None, "share_of_step": walk_ms / ms_step, "kernels": kern},
        "cpu_baseline": {"value": cpu_n / cpu_dt, "unit": UNIT, "cores": cores, "kind": "port",
                         "sample": f"{cpu_n} replies in {cpu_dt:.1f} s over {cores} processes (oracle/port.py reply_output)"},
    }
    sys.stdout.flush()
    os.write(real_stdout, (json.dumps(line) + "\n").encode())
    torch.cuda.synchronize()
    del stream
    eng.close()
    teardown(world)


def _cpu_mixed_worker(chunk):
    return _cpu_worker(chunk)


def run_mixed(args, rank, world, local_rank, dev, real_stdout, all_cpus=None) -> None:
    """BASELINE.json configs[4]: mixed-size event stream (128 B - 64 KB JSON: multi-turn histories with escapes and multi-byte
    UTF-8), callbacks spread over 256 subscribe_topics; the tool-node path (decode -> run -> publish plan -> encode -> route)."""
    import multiprocessing as mp
    import numpy as np
    import torch
    from calfkit import synth
    from calfkit.engine import BatchEngine, ToolTemplate
    n = args.events if args.events != 1_000_000 else 65536
    base = synth.mixed_events(4096, seed=5000 + rank, hi=65536, n_agents=256)
    recs = [base[i % len(base)] for i in range(n)]
    batch = synth.pack(recs)
    in_bytes = int(batch.data.nbytes)
    topics = [f"agent_{k:03d}.input" for k in range(256)] + ["tool.get_weather.input", "tool.get_weather.output"]
    eng = BatchEngine(local_rank, max_records=n, max_in_bytes=in_bytes + 4096)
    eng.register_topics(topics, num_partitions=NUM_PARTITIONS)
    eng.set_tool_node("tool.get_weather.output", ToolTemplate.from_format(TOOL_FMT))
    eng.set_bucketing(True)            # sizes from 128 B to 64 KB in one batch: bucket by length before the walk
    d_in = torch.from_numpy(batch.data.copy()).to(dev)
    d_off = torch.from_numpy(batch.offsets.copy()).to(dev)
    stream = torch.cuda.ExternalStream(eng.stream_ptr(), device=dev)

    def step():
        eng.submit_device(d_in, d_off, n)
        eng.tool_plan()

    for _ in range(args.warmup):
        step()
    eng.sync()
    eng.profile(True)
    sampler = ClockSampler(local_rank)
    sampler.start()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    l0 = eng.launch_count()
    ev0.record(stream)
    for _ in range(args.steps):
        step()
    ev1.record(stream)
    torch.cuda.synchronize()
    sampler.stop_flag = True
    gpu_launches = eng.launch_count() - l0
    ms_step = ev0.elapsed_time(ev1) / args.steps
    prof = eng.profile_read()
    eng.profile(False)
    out_bytes, npay, npub = eng.out_size()
    value = world * n / (ms_step / 1e3)
    if args.dump_outputs and rank == 0:
        dump_outputs(eng, args.dump_outputs)
    from calfkit.engine.lane import Arena, LanePipeline
    pipe = LanePipeline(local_rank, lambda e_: (e_.register_topics(topics, num_partitions=NUM_PARTITIONS),
                                                e_.set_tool_node("tool.get_weather.output", ToolTemplate.from_format(TOOL_FMT)), e_.set_bucketing(True)),
                        lanes=3, max_records=n, max_in_bytes=in_bytes + 4096)
    h_in = torch.from_numpy(batch.data.copy()).pin_memory()
    h_off = torch.from_numpy(batch.offsets.copy()).pin_memory()
    arena = Arena(h_in.numpy(), h_off.numpy())
    d2h, e2e_steps = 0, args.steps
    for k in range(3 + e2e_steps):
        if k == 3:
            for pb in pipe.drain():
                pb.release()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        pb = pipe.push(arena)
        if pb is not None:
            pb.release()
    for pb in pipe.drain():
        d2h = max(d2h, max(l_.d2h_bytes for l_ in pipe.lanes))
        pb.release()
    torch.cuda.synchronize()
    e2e_ms = (time.perf_counter() - t0) * 1e3 / e2e_steps
    pipe.close()
    cols = eng.columns()
    peak, _peak_src = hbm_peak_gbs()
    kern = {k: {"ms_per_step": ms / args.steps, "launches_per_step": c / args.steps} for k, (ms, c) in prof.items() if c}
    # the decode of this workload is three kernels: warp pre-scan of the long records (walk_long), the thread-per-record
    # walk (walk; with bucketing on, the sort passes are timed with it), one thread per history message (walk_elems)
    walk_ms = sum(kern[k]["ms_per_step"] for k in ("walk", "walk_long", "walk_elems") if k in kern)
    from calfkit.engine._lib import COL as _COL, NUM_COLS as _NC
    algo_walk = in_bytes + 8 * (n + 1) + 4 * (_NC - 10) * n
    from oracle import port
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import tools_def
    small = synth.pack(recs[:128])
    chk = eng.run_tool_batch(small.data, small.offsets)
    node = port.ToolNode.of(tools_def.get_weather)
    parity_ok = [(p.topic, p.key, p.payload) for p in chk.publishes()] == \
        [(tp, k, pl) for r in recs[:128] for (tp, k, _c, pl) in port.tool_node_event(node, r)]
    cores = os.cpu_count() or 1
    sample = recs[: max(cores * 16, 256)]
    if all_cpus:
        os.sched_setaffinity(0, all_cpus)
    rpool = ReferencePool(cores)
    rpool.run(sample[: max(cores, 16)])
    cpu_value, cpu_dt, cpu_n = rpool.run(sample)
    cpu_kind, cpu_desc = rpool.kind, rpool.describe()
    rpool.close()
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_step,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": dict(bench_config(args, world), events_per_gpu_per_step=n, topics=len(topics)),
        "workload_stats": {"record_bytes_mean": in_bytes / n, "record_bytes_max": int(np.diff(batch.offsets).max()), "in_gb_per_step": in_bytes / 1e9,
                           "input_gbs": in_bytes / ms_step / 1e6, "ok_fraction": float((cols[_COL["STATUS"]] == 0).mean()),
                           "parity_spot_check_128": parity_ok, "out_bytes_per_event": out_bytes / n},
        "clocks": sampler.summary(),
        "e2e": {"value": world * n / (e2e_ms / 1e3), "unit": UNIT, "h2d_bytes_per_step": in_bytes + 8 * (n + 1), "d2h_bytes_per_step": d2h,
                "ms_per_step": e2e_ms, "steps": e2e_steps, "api": "calfkit.engine.lane.LanePipeline.push(pinned Arena) -> PublishBatch (3 lanes)"},
        "gpu_launches": gpu_launches,
        "roofline": {"kernel": "decode = ck_walk_long_kernel (pre-scan) + ck_walk_kernel + ck_walk_elems_kernel", "bound": "hbm",
                     "achieved": algo_walk / walk_ms / 1e6, "peak": peak, "unit": "GB/s",
                     "frac": algo_walk / walk_ms / 1e6 / peak, "traffic": None, "share_of_step": walk_ms / ms_step, "kernels": kern,
                     "pipeline": {"algo_bytes_per_event": (in_bytes + out_bytes) / n, "achieved": (in_bytes + out_bytes) / ms_step / 1e6,
                                  "frac": (in_bytes + out_bytes) / ms_step / 1e6 / peak}},
        "cpu_baseline": {"value": cpu_value, "unit": UNIT, "cores": cores, "kind": cpu_kind,
                         "sample": f"{cpu_n} events of the same batch in {cpu_dt:.1f} s over {cores} processes; " + cpu_desc},
    }
    sys.stdout.flush()
    os.write(real_stdout, (json.dumps(line) + "\n").encode())
    torch.cuda.synchronize()
    del stream
    eng.close()
    teardown(world)


# ------------------------------------------------------------------------------------------------ GPU arm
def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10, help="timed steps of every leg (device-resident and end to end)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--events", type=int, default=1_000_000, help="events per GPU per step (config 2: 1M)")
    ap.add_argument("--cross", type=float, default=0.125, help="fraction of records on a foreign partition (N > 1)")
    ap.add_argument("--cpu-sample", type=int, default=0, help="events for the cpu_baseline leg (0 = auto)")
    ap.add_argument("--workload", default="tool_event_1k", choices=["tool_event_1k", "fanout", "reply", "mixed"],
                    help="tool_event_1k = BASELINE.json configs[1] (the headline); fanout = configs[2]: 1 Agent -> 64 tools")
    ap.add_argument("--fanout", type=int, default=64)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last one computed (rank 0) as DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    if args.impl == "reference":
        run_reference(args, rank, world)
        return
    # stdout carries exactly ONE JSON line: anything a library prints to fd 1 (NCCL's version banner ...) goes to stderr
    real_stdout = os.dup(1)
    os.dup2(2, 1)
    if args.warmup < 3:
        args.warmup = 3

    import numpy as np
    import torch
    import torch.distributed as dist
    from calfkit import synth
    from calfkit.engine import BatchEngine, ToolTemplate
    from calfkit.engine._lib import COL, PUB_DTYPE

    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    # host threads + pinned staging buffers next to this GPU's PCIe root (one process per GPU; restored for the CPU leg)
    from calfkit.engine.batch import bind_host_to_gpu
    all_cpus = os.sched_getaffinity(0)
    numa_cpus = bind_host_to_gpu(local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")     # NCCL's version banner / logs must not land on stdout: one JSON line only
        opts = dist.ProcessGroupNCCL.Options()
        opts.is_high_priority_stream = True          # the per-step barriers must not queue behind the big kernels
        dist.init_process_group("nccl", device_id=dev, pg_options=opts)

    if args.workload == "fanout":
        run_fanout(args, rank, world, local_rank, dev, real_stdout, all_cpus)
        return
    if args.workload == "reply":
        run_reply(args, rank, world, local_rank, dev, real_stdout, all_cpus)
        return
    if args.workload == "mixed":
        run_mixed(args, rank, world, local_rank, dev, real_stdout, all_cpus)
        return
    n = args.events
    recs = synth.tool_events(n, seed=1000 + rank)
    batch = synth.pack(recs)
    del recs
    in_bytes = int(batch.data.nbytes)
    topics = ["tool.get_weather.input", "tool.get_weather.output", "weather_agent.input"]
    import ctypes as C
    from calfkit.engine.exchange import PeerExchange
    launches = [0]

    all_lanes = []

    class Lane:
        """one BatchEngine (= one CUDA stream + its HBM buffers) with torch views of its result tables and
        a pinned host landing buffer; two lanes ping-pong in the end-to-end loop (double buffering)"""
        def __init__(self):
            all_lanes.append(self)
            self.eng = eng = BatchEngine(local_rank, max_records=n, max_in_bytes=in_bytes + 4096)
            eng.register_topics(topics, num_partitions=NUM_PARTITIONS)
            eng.set_tool_node("tool.get_weather.output", ToolTemplate.from_format(TOOL_FMT))
            self.stream = torch.cuda.ExternalStream(eng.stream_ptr(), device=dev)
            bufs = eng.device_buffers()
            p_pubs, p_len, p_desc = C.c_void_p(), C.c_void_p(), C.c_void_p()
            eng.lib.ck_device_buffers2(eng.h, C.byref(p_pubs), C.byref(p_len), C.byref(p_desc))
            self.t_pubs = torch.as_tensor(CudaArray(p_pubs.value, (2 * n, 8), "<i4"), device=dev)
            self.t_out_off = torch.as_tensor(CudaArray(bufs["out_off"], (n + 1,), "<i8"), device=dev)
            self.t_out_len = torch.as_tensor(CudaArray(p_len.value, (n,), "<i4"), device=dev)
            self.out_cap = eng.max_out
            self.t_out = torch.as_tensor(CudaArray(bufs["out"], (self.out_cap,), "|u1"), device=dev)
            self.px, self.step_no = None, 0
            if world > 1:
                # receive regions for what the other ranks forward here: one per source, sized for 2 x the expected share
                fwd = int(n * min(1.0, args.cross * 2 + 0.05) / (world - 1)) + 1024
                self.px = PeerExchange(eng, rank, world, max_fwd=fwd, data_cap=fwd * (int(in_bytes / n) + 64))
                rp, rs, rmf, rdc = C.c_void_p(), C.c_uint64(), C.c_uint32(), C.c_uint64()
                eng.lib.ck_recv_info(eng.h, C.byref(rp), C.byref(rs), C.byref(rmf), C.byref(rdc))
                self.region_stride, self.region_hdr = rs.value, 64 + 16 * rmf.value
                self.t_recv = torch.as_tensor(CudaArray(rp.value, (world * rs.value,), "|u1"), device=dev)
                self.h_recv = torch.empty(world * rs.value, dtype=torch.uint8).pin_memory()
            self.h_out = torch.empty(self.out_cap, dtype=torch.uint8).pin_memory()
            self.h_out_np = self.h_out.numpy()
            # pinned landing buffers for the offsets / lengths / publish table as well
            self.h_off = torch.empty(n + 1, dtype=torch.int64).pin_memory().numpy()
            self.h_len = torch.empty(n, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
            self.h_pubs = torch.empty(2 * n * PUB_DTYPE.itemsize, dtype=torch.uint8).pin_memory().numpy().view(PUB_DTYPE)
            self.d2h = 0
            self.rbytes = 0

        def close(self):
            # every torch object that touched this engine's stream goes first (the caching allocators record an event on a
            # tensor's streams when it is freed: the stream must still exist), then the engine (stream + HBM buffers)
            import gc
            self.t_pubs = self.t_out_off = self.t_out_len = self.t_out = self.t_recv = self.h_recv = None
            self.h_out = self.h_out_np = self.h_off = self.h_len = self.h_pubs = None
            self.px = None
            gc.collect()
            torch.cuda.synchronize()
            self.stream = None
            self.eng.close()

        def exchange(self):
            """forward keyed payloads whose partition is owned by another GPU: the library's kernels plan, pack and store
            them straight into the owners' receive regions over NVLink (no host synchronisation); two 4-byte barriers"""
            self.step_no += 1
            with torch.cuda.stream(self.stream):
                self.px.send(self.step_no)

        def enqueue_device(self, d_in, d_off):
            self.eng.submit_device(d_in, d_off, n)
            self.eng.tool_plan()
            launches[0] += 7            # walk, plan, 3 x scan, emit, route

        def enqueue_host(self, h_in_np, h_off_np):
            self.eng.submit(h_in_np, h_off_np)          # asynchronous H2D of the batch from pinned memory + decode
            self.eng.tool_plan()

        def exchange_host(self):
            """N > 1: forward foreign-partition payloads and land what this rank received in pinned memory (headers first: they
            say how many bytes each source sent).  Called after the other lane's D2H so that the wait does not stall the copies."""
            if world > 1:
                self.exchange()
                with torch.cuda.stream(self.stream):
                    hdrs = self.t_recv.view(world, self.region_stride)[:, :32].contiguous().cpu().view(torch.int64)    # waits for the closing barrier
                    self.rbytes = 0
                    for s_ in range(world):
                        if s_ == rank:
                            continue
                        if int(hdrs[s_, 1]) >> 32:
                            raise RuntimeError("exchange region overflow: raise max_fwd / data_cap")
                        nbytes = self.region_hdr + int(hdrs[s_, 2])
                        a = s_ * self.region_stride
                        self.h_recv[a:a + nbytes].copy_(self.t_recv[a:a + nbytes], non_blocking=True)
                        self.rbytes += nbytes

        def fetch_host(self):
            out, off, ln, pubs = self.eng._fetch(out_buf=self.h_out_np, off_buf=self.h_off, len_buf=self.h_len,
                                                 pubs_buf=self.h_pubs)   # D2H: payloads, offsets, lengths, publishes (waits)
            self.d2h = int(out.nbytes + off.nbytes + ln.nbytes + pubs.nbytes + self.rbytes)

    lane = Lane()
    eng = lane.eng
    if world > 1:
        eng.submit(batch.data, batch.offsets)
        corr_off = eng.columns()[COL["CORR_OFF"]]
        batch = place_on_partitions(batch, corr_off, rank, world, args.cross, seed=2000 + rank)

    h_in = torch.from_numpy(batch.data.copy()).pin_memory()
    h_off = torch.from_numpy(batch.offsets.copy()).pin_memory()
    d_in = h_in.to(dev)
    d_off = h_off.to(dev)
    stream = lane.stream

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- device-resident timing ------------------------------------------------------------------
    # N == 1: one lane, back-to-back steps.  N > 1: two lanes alternate so that the (latency-bound: host-side
    # split sizes + three small collectives) cross-partition exchange of step k overlaps the kernels of
    # step k+1 on the other lane's stream.
    lanes = [lane, Lane()] if world > 1 else [lane]

    def run_device(k_steps):
        if world == 1:
            for _ in range(k_steps):
                lane.enqueue_device(d_in, d_off)
            return
        lanes[0].enqueue_device(d_in, d_off)
        for k in range(1, k_steps):
            lanes[k % 2].enqueue_device(d_in, d_off)
            lanes[(k - 1) % 2].exchange()
        lanes[(k_steps - 1) % 2].exchange()

    run_device(args.warmup)
    torch.cuda.synchronize()
    eng.profile(True)
    sampler = ClockSampler(local_rank)
    barrier()
    sampler.start()
    ev0 = torch.cuda.Event(enable_timing=True)
    ev_end = [torch.cuda.Event(enable_timing=True) for _ in lanes]
    launch0 = sum(ln_.eng.launch_count() for ln_ in lanes)
    for ln_ in lanes[1:]:
        ln_.stream.wait_stream(lanes[0].stream)
    ev0.record(lanes[0].stream)
    for ln_ in lanes[1:]:
        ln_.stream.wait_event(ev0)                       # no lane starts before the start event
    run_device(args.steps)
    for e_, ln_ in zip(ev_end, lanes):
        e_.record(ln_.stream)
    barrier()
    ms_total = max(ev0.elapsed_time(e_) for e_ in ev_end)
    sampler.stop_flag = True
    prof = eng.profile_read()
    eng.profile(False)
    gpu_launches = sum(ln_.eng.launch_count() for ln_ in lanes) - launch0     # counted by the library at every kernel launch
    out_bytes, npay, npub = eng.out_size()
    out_payload_bytes = int(lane.t_out_len.to(torch.int64).sum().item())
    cols = eng.columns()
    ok_frac = float((cols[COL["STATUS"]] == 0).mean())
    t = torch.tensor([ms_total], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_total = float(t.item())
    ms_step = ms_total / args.steps
    value = world * n / (ms_step / 1e3)
    if args.dump_outputs and rank == 0:
        dump_outputs(lanes[(args.steps - 1) % len(lanes)].eng, args.dump_outputs)

    # ---- end to end (host buffers), pipelined over several engines (3 at N = 1, 2 at N > 1) -----------------
    # step k: lane k%2 takes the batch from pinned host memory (H2D + all kernels, asynchronous) while the
    # previous step's results are copied back from the other lane (D2H + wait): the two PCIe directions
    # and the kernels overlap, exactly as a worker consuming a stream of batches would run it.
    if world == 1:
        lanes = [lane, Lane(), Lane()]          # triple buffering: the D2H of step k-2 never waits for kernels
    h_in_np, h_off_np = h_in.numpy(), h_off.numpy()
    e2e_steps = args.steps

    def run_e2e(k_steps):
        if world == 1:
            # step k: lane k%3 takes the batch (H2D + kernels, asynchronous); the results of step k-2 — whose kernels
            # finished a step ago — are copied back at the same time, so both PCIe directions stay busy
            L = len(lanes)
            for k in range(k_steps):
                lanes[k % L].enqueue_host(h_in_np, h_off_np)
                if k >= L - 1:
                    lanes[(k - (L - 1)) % L].fetch_host()
            for k in range(max(0, k_steps - (L - 1)), k_steps):
                lanes[k % L].fetch_host()
            return
        lanes[0].enqueue_host(h_in_np, h_off_np)
        lanes[0].exchange_host()
        for k in range(1, k_steps):
            lanes[k % 2].enqueue_host(h_in_np, h_off_np)
            lanes[(k - 1) % 2].fetch_host()
            lanes[k % 2].exchange_host()
        lanes[(k_steps - 1) % 2].fetch_host()

    run_e2e(4)
    barrier()
    t0 = time.perf_counter()
    run_e2e(e2e_steps)
    torch.cuda.synchronize()
    wall_ms = (time.perf_counter() - t0) * 1e3
    barrier()
    t = torch.tensor([wall_ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    e2e_ms = float(t[0].item()) / e2e_steps
    e2e_value = world * n / (e2e_ms / 1e3)
    d2h_bytes = [lanes[0].d2h]

    # ---- host-copy ceiling: the same bytes per step as plain concurrent H2D + D2H copies, no kernels, all ranks at once -------
    c_h2d = torch.empty(in_bytes, dtype=torch.uint8).pin_memory()
    c_d2h = torch.empty(lanes[0].d2h or in_bytes, dtype=torch.uint8).pin_memory()
    c_din = torch.empty(in_bytes, dtype=torch.uint8, device=dev)
    c_dout = torch.empty(c_d2h.numel(), dtype=torch.uint8, device=dev)
    s_up, s_dn = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
    c_steps = 6
    for k_ in range(2 + c_steps):
        if k_ == 2:
            barrier()
            t0 = time.perf_counter()
        with torch.cuda.stream(s_up):
            c_din.copy_(c_h2d, non_blocking=True)
        with torch.cuda.stream(s_dn):
            c_d2h.copy_(c_dout, non_blocking=True)
    torch.cuda.synchronize()
    c_ms = (time.perf_counter() - t0) * 1e3
    barrier()
    tc_ = torch.tensor([c_ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(tc_, op=dist.ReduceOp.MAX)
    c_ms = float(tc_.item()) / c_steps
    ceiling = {"events_per_s": world * n / (c_ms / 1e3), "ms_per_step": c_ms, "h2d_gbs_per_gpu": in_bytes / c_ms / 1e6,
               "d2h_gbs_per_gpu": c_d2h.numel() / c_ms / 1e6,
               "what": "plain cudaMemcpyAsync of one step's bytes in both directions at once from/to pinned host memory on every rank, no kernels"}
    del c_h2d, c_d2h, c_din, c_dout, s_up, s_dn

    # ---- N > 1: the bytes each rank RECEIVED against what their senders planned (outside all timed regions) ---------------
    x_parity = None
    if world > 1:
        ln0 = lanes[0]
        ln0.eng.submit(h_in_np, h_off_np)
        ln0.eng.tool_plan()
        ln0.step_no += 1
        with torch.cuda.stream(ln0.stream):
            ln0.px.send(ln0.step_no)
        recv = ln0.px.received(ln0.step_no)
        out_b, off_b, len_b, pubs_b = ln0.eng._fetch()
        keyed = (pubs_b["payload"] != 0xFFFFFFFF) & (pubs_b["has_key"] == 1)
        mine = {}
        for d_ in range(world):
            if d_ != rank:
                idx_ = np.nonzero(keyed & (pubs_b["partition"] % world == d_))[0]
                mine[d_] = (len(idx_), [out_b[off_b[p_]:off_b[p_] + len_b[p_]].tobytes() for p_ in pubs_b["payload"][idx_[:64]]])
        allm = [None] * world
        dist.all_gather_object(allm, mine)
        okx = True
        for src_, meta_, data_ in recv:
            cnt_, first_ = allm[src_][rank]
            okx = okx and cnt_ == len(meta_) and PeerExchange.payloads(meta_[:64], data_) == first_ \
                and bool(((meta_["partition"] % world) == rank).all())
        tx = torch.tensor([1 if okx else 0], device=dev)
        dist.all_reduce(tx, op=dist.ReduceOp.MIN)
        x_parity = bool(tx.item())

    # ---- end to end through the product API: Worker.run() over a batch-native broker -----------------------------------
    # the same pinned batch is produced `w_steps` times to the node's input topic; Worker.run polls it as arenas, drives its
    # own LanePipeline (H2D + kernels of step k overlap the D2H of step k-1 and the host-side produce of step k-2) and hands
    # publish batches to the broker, where two sinks (the agent's topic and the node's publish_topic) count what a Kafka
    # producer would send.  Timed with the host clock around run(until_idle=True), synchronised on both sides.
    import asyncio
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import tools_def as _td
    from calfkit import Client, Worker, agent_tool
    from calfkit.engine.lane import Arena
    w_node = agent_tool(_td.get_weather, device_template=TOOL_FMT)
    w_client = Client.connect("localhost")
    w_cnt = {"pubs": 0, "payload_bytes": 0}

    def w_sink(b, idx):
        w_cnt["pubs"] += len(idx)
    w_client.broker.sink("weather_agent.input", w_sink)
    w_client.broker.sink("tool.get_weather.output", w_sink)
    worker = Worker(w_client, nodes=[w_node], device=local_rank, batch_records=n, batch_bytes=in_bytes + 4096, lanes=3,
                    route_topics=["weather_agent.input"])
    w_arena = Arena(h_in_np[:in_bytes], h_off_np)
    for _ in range(3):
        w_client.broker.produce_arena("tool.get_weather.input", w_arena)
    asyncio.run(worker.run(until_idle=True))
    w_steps = args.steps
    w_cnt["pubs"] = 0
    for _ in range(w_steps):
        w_client.broker.produce_arena("tool.get_weather.input", w_arena)
    w_l0 = sum(p_.launch_count() for p_ in worker._pipes.values())
    barrier()
    t0 = time.perf_counter()
    asyncio.run(worker.run(until_idle=True))
    torch.cuda.synchronize()
    w_ms = (time.perf_counter() - t0) * 1e3
    barrier()
    t = torch.tensor([w_ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    w_ms = float(t[0].item()) / w_steps
    w_value = world * n / (w_ms / 1e3)
    w_launches = sum(p_.launch_count() for p_ in worker._pipes.values()) - w_l0
    w_d2h = max(l_.d2h_bytes for p_ in worker._pipes.values() for l_ in p_.lanes)
    tw = torch.tensor([w_cnt["pubs"], worker.stats["rejected"]], dtype=torch.int64, device=dev)
    if world > 1:
        dist.all_reduce(tw)                      # a forwarded publish is produced (and counted) by the rank that owns its partition
    w_ok = int(tw[0].item()) == world * 2 * n * w_steps and int(tw[1].item()) == 0
    worker.close()

    def shutdown():
        # orderly teardown: drop every torch view of library-owned device memory, destroy the engines (streams +
        # HBM buffers) while the CUDA context is alive, leave the process group, and return normally so that
        # interpreter exit hooks (the driver's loaded-.so record) run
        sys.stdout.flush()
        sys.stderr.flush()
        torch.cuda.synchronize()
        for ln_ in all_lanes:
            ln_.close()
        teardown(world)

    if rank != 0:
        shutdown()
        return

    # ---- roofline of the dominant kernel -------------------------------------------------------------
    peak, peak_src = hbm_peak_gbs()
    ncols_walk = COL["NOUT"]
    algo = {   # algorithmic bytes per launch (DESIGN.md §kernels)
        "walk": in_bytes + 8 * (n + 1) + 4 * ncols_walk * n,
        "plan": 4 * 24 * n + 160 * n + 2 * 32 * n + 4 * n,
        "scan": 3 * 4 * n + 8 * n,
        "emit": 2 * out_payload_bytes + 160 * n + 8 * n,
        "route": 2 * 2 * 32 * n,
    }
    kern = {}
    for k, (ms, cnt) in prof.items():
        if cnt and k in algo:
            kern[k] = {"ms_per_launch": ms / cnt, "launches": cnt, "algo_bytes": algo[k],
                       "gbs": algo[k] / (ms / cnt) / 1e6 if k != "scan" else None}
    kern_step_ms = sum(v[0] / v[1] for v in prof.values() if v[1])        # one launch of each per step
    dom = max((k for k in kern if k != "scan"), key=lambda k: kern[k]["ms_per_launch"])
    traffic = None
    tpath = os.path.join(ROOT, "profiles", "traffic.json")
    if os.path.exists(tpath):
        tj = json.load(open(tpath))
        if dom in tj:
            traffic = tj[dom]["dram_bytes_per_record"] * n
    achieved = kern[dom]["gbs"]
    roofline = {"kernel": f"ck_{dom}_kernel", "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s",
                "frac": achieved / peak, "traffic": traffic, "peak_source": peak_src,
                "share_of_step": kern[dom]["ms_per_launch"] / ms_step,
                "pipeline": {"algo_bytes_per_event": (in_bytes + out_payload_bytes) / n,
                             "achieved": (in_bytes + out_payload_bytes) / ms_step / 1e6,
                             "frac": (in_bytes + out_payload_bytes) / ms_step / 1e6 / peak},
                "kernels": kern, "sum_kernel_ms_per_step": kern_step_ms}

    # ---- CPU baseline: the reference's own code on a bounded sample of the same batch, all host cores -------------
    os.sched_setaffinity(0, all_cpus)
    cores = os.cpu_count() or 1
    sample_n = args.cpu_sample or max(cores * 1500, 20000)       # ~10-30 s of CPU work over all cores
    sample = [batch.record(i) for i in range(min(sample_n, n))]
    rpool = ReferencePool(cores)
    rpool.run(sample[: max(cores * 8, 64)])
    cpu_value, cpu_dt, cpu_n = rpool.run(sample)
    cpu_kind, cpu_desc = rpool.kind, rpool.describe()
    rpool.close()
    try:                                                                # second figures: the oracle port, and one core
        port_value, _dtp, _np = cpu_arm(sample, cores, start="spawn")
        one = ReferencePool(1)
        one.run(sample[:64])
        one_core_value, _dt1, _n1 = one.run(sample[:2000])
        one.close()
    except Exception:  # noqa: BLE001  (never let the extra figures cost the bench line)
        port_value = one_core_value = None
    # parity spot check against the oracle on the same bytes (byte-exact), outside all timed regions
    from oracle import port
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import tools_def
    small = synth.pack(sample[:256])
    chk = eng.run_tool_batch(small.data, small.offsets)
    node = port.ToolNode.of(tools_def.get_weather)
    pubs = [(p.topic, p.key, p.payload) for p in chk.publishes()]
    want = [(tp, k, pl) for r in sample[:256] for (tp, k, _c, pl) in port.tool_node_event(node, r)]
    parity_ok = pubs == want

    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8",
        "data": "synthetic",
        "config": bench_config(args, world),
        "workload_stats": {"record_bytes_mean": in_bytes / n, "out_bytes_mean": out_payload_bytes / max(npay, 1), "publishes_per_event": 2,
                           "accepted_fraction": ok_frac, "parity_spot_check_256": parity_ok, "in_gb_per_step": in_bytes / 1e9,
                           "exchange_parity": x_parity},
        "clocks": sampler.summary(),
        "e2e": {"value": w_value, "unit": UNIT, "h2d_bytes_per_step": in_bytes + 8 * (n + 1), "d2h_bytes_per_step": w_d2h,
                "ms_per_step": w_ms, "steps": w_steps, "gpu_launches": w_launches, "all_publishes_seen_by_sinks": w_ok,
                "api": "calfkit.Worker.run(until_idle=True): MemoryBroker.poll_arena (pinned batch) -> LanePipeline (3 lanes) -> "
                       "MemoryBroker.produce_publishes -> per-topic sinks; N > 1: one Worker per GPU, keyed publishes forwarded to the rank that owns their partition inside Worker.run",
                "timing": "host wall clock around Worker.run, synchronised on both sides, max over ranks",
                "ceiling": ceiling, "frac_of_ceiling": w_value / ceiling["events_per_s"],
                "engine_level": {"value": e2e_value, "ms_per_step": e2e_ms, "steps": e2e_steps, "d2h_bytes_per_step": d2h_bytes[0],
                                 "api": "BatchEngine.submit(pinned host) + tool_plan + fetch(pinned host), %d engines pipelined%s"
                                        % (len(lanes), " + cross-partition exchange" if world > 1 else "")}},
        "gpu_launches": gpu_launches,
        "roofline": roofline,
        "cpu_baseline": {"value": cpu_value, "unit": UNIT, "cores": cores, "kind": cpu_kind,
                         "sample": f"{cpu_n} events of the same batch in {cpu_dt:.1f} s over {cores} processes; " + cpu_desc,
                         "oracle_port": {"value": port_value, "unit": UNIT, "cores": cores, "sample": "same events, oracle/port.py"},
                         "one_core": {"value": one_core_value, "unit": UNIT, "sample": "2000 events, 1 process, same code"}},
    }
    sys.stdout.flush()
    os.write(real_stdout, (json.dumps(line) + "\n").encode())
    shutdown()


if __name__ == "__main__":
    main()
