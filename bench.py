#!/usr/bin/env python3
"""bench.py -- CheckResources decisions/sec of the H100 evaluator (BASELINE.json metric).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--workload C2] [--impl ours|reference] [--dump-outputs DIR]
    torchrun --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...       (N > 1, one rank per GPU)

A *step* is `batches_per_step` passes of the hot path (rule-table scan + CEL condition evaluation), each over one
batch of synthetic requests of the workload; the count is chosen once, after warm-up, so that a step is at least
~10 ms of device work (reported in `config`).  Default workload: C3 of SURVEY.md 8(d) = BASELINE.json configs[2], the
largest single-GPU configuration (100 scoped resource policies, 3-level scope chains, 20 CEL conditions with string /
list operations, 2^24 requests x 8 actions per batch).  At --gpus 8 the same command is configs[3] ("C4": the C3 table,
2^27 requests sharded over 8 GPUs).  Weak scaling: every rank evaluates its own shard of the request stream (no
data-path collective); the packed decision bitmaps are exchanged over NVLink so that every rank holds the whole result.
A C2 (configs[1]) measurement rides along as `secondary` at N = 1.

  value     whole-job decisions/s with the request columns already resident in HBM (CUDA events, max over
            ranks; successive steps rotate over distinct batches whose total footprint exceeds L2)
  e2e       the same metric through the host-buffer C-ABI call cgpu_check (pinned host columns -> H2D ->
            kernel -> D2H -> effect bytes), i.e. what engine.Check would pay per call
  roofline  algorithmic bytes / launch (SURVEY.md 8(d): C3 197 B, C2 73 B per request) over the mean kernel duration vs the
            measured HBM copy bandwidth (MEASURED_PEAKS.json; without it the H100 SXM data sheet's 3.35 TB/s)
  cpu_baseline  oracle/c/check_ref.c (a plain-C port of the reference algorithm) on all host cores

--dump-outputs DIR writes, after the timed steps, the decisions of the last step as float32 .npy files (1 = ALLOW,
2 = DENY; a fixed, seeded sample of requests of every batch that step evaluated) and the sampled request indices, at
most about 48 MB in all.  Inputs are generated from fixed seeds, so two builds run with the same arguments can be
compared output for output.

--impl reference times that CPU port alone (the Go toolchain needed for the reference's own engine is not
in this image; see DESIGN.md).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "checkresources_decisions_per_sec"
UNIT = "decisions/s"
NOW_NS = 1_700_000_000_000_000_000


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            with open(p) as f:
                return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
        except Exception:
            pass
    return 3350.0, "fallback (H100 SXM data sheet: 3.35 TB/s HBM3; not a measured figure)"


class ClockSampler:
    """Samples nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index=0):
        self.gpu = gpu_index
        self.samples = []
        self._stop = threading.Event()
        self._t = None

    def _run_nvml(self) -> bool:
        """NVML in-process: ~1 ms per sample (an nvidia-smi process takes ~100 ms, longer than a short timed region)."""
        try:
            import pynvml
            pynvml.nvmlInit()
            idx = self.gpu
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            if vis:
                ids = [x.strip() for x in vis.split(",") if x.strip()]
                if self.gpu < len(ids) and ids[self.gpu].isdigit():
                    idx = int(ids[self.gpu])
            h = pynvml.nvmlDeviceGetHandleByIndex(idx)
            mx = str(pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM))
            bits = [pynvml.nvmlClocksThrottleReasonHwSlowdown, pynvml.nvmlClocksThrottleReasonHwThermalSlowdown,
                    pynvml.nvmlClocksThrottleReasonSwThermalSlowdown, pynvml.nvmlClocksThrottleReasonSwPowerCap]
            pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)
        except Exception:  # noqa: BLE001 -- no NVML: fall back to nvidia-smi
            return False
        while not self._stop.is_set():
            try:
                r = pynvml.nvmlDeviceGetCurrentClocksThrottleReasons(h)
                self.samples.append([str(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)), mx, "0"] +
                                    ["Active" if r & b else "Not Active" for b in bits])
            except Exception:  # noqa: BLE001
                pass
            self._stop.wait(0.002)
        return True

    def _run(self):
        if self._run_nvml():
            return
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                      "-i", str(self.gpu)], capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.samples.append([x.strip() for x in out.split(",")])
            except Exception:
                pass
            self._stop.wait(0.1)

    def __enter__(self):
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        t0 = time.time()
        while not self.samples and time.time() - t0 < 3.0:   # sampler initialised (NVML / first nvidia-smi) before the timed region starts
            time.sleep(0.002)
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join(timeout=6)

    def summary(self):
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for s in self.samples:
            try:
                sm.append(float(s[0]))
                mx.append(float(s[1]))
                for nm, v in zip(names, s[3:7]):
                    if v.lower().startswith("active"):
                        reasons.add(nm)
            except Exception:
                continue
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(mx), "reasons": sorted(reasons), "samples": len(sm)}


def get_workload(name):
    import workloads as W
    return W.WORKLOADS[name]()


def _serialized_chunk(job):
    """(worker process) serialized enginev1.CheckInput messages of requests [start, start + n) of a workload's stream"""
    name, n, start = job
    from cerbos_b200 import wire
    import workloads as W
    w = W.WORKLOADS[name]()
    return [wire.check_input(x) for x in w.inputs(w.fields(n, start=start), range(n))]


def native_columns(w, n, start, blob):
    """Columns of a workload without a vectorised column builder (C5), at bench scale: worker processes generate and
    serialize the requests (the Python part), the native encoder (cgpu_encode, host threads) builds the batch."""
    import multiprocessing as mp
    from concurrent.futures import ProcessPoolExecutor
    from cerbos_b200 import capi
    from cerbos_b200.encode import Batch, passes_for
    chunk = 4096
    jobs = [(w.name, min(chunk, n - o), start + o) for o in range(0, n, chunk)]
    if len(jobs) > 1:
        with ProcessPoolExecutor(max_workers=min(48, os.cpu_count() or 1, len(jobs)), mp_context=mp.get_context("spawn")) as pool:
            parts = list(pool.map(_serialized_chunk, jobs))
    else:
        parts = [_serialized_chunk(j) for j in jobs]
    msgs = [m for p in parts for m in p]
    ne = capi.NativeEncoder(blob)
    eb = ne.encode(msgs)
    raw = eb.columns()
    K = int(eb.batch().max_actions)
    eb.free()
    ne.close()
    hdr1_t = np.dtype([("rv", "<u2"), ("pv", "<u2"), ("aset", "<u4")])
    rc = raw[2].nbytes // (4 * n)
    cols = [raw[0].view(np.uint32).reshape(n, 4), raw[1].view(hdr1_t), raw[2].view(np.uint32).reshape(rc, n), raw[3].view(np.uint64).reshape(-1, n),
            raw[4].view(np.uint64), raw[5].view(np.uint32), raw[6], raw[7].view(np.uint32), raw[8].view(np.uint32), raw[9].view(np.uint32),
            raw[10].view(np.uint64), raw[11].view(np.uint64)]
    kc, n_pass = passes_for(K, rc)
    return Batch(n, K, rc, cols, None, n_pass, kc)


def shard_columns(w, n, shard, enc, blob=None):
    """Columns of requests [shard*n, (shard+1)*n) of the workload's stream (built in parallel chunks)."""
    import workloads as W
    if w.name in ("C2", "C3", "C5"):
        return W.columns_parallel(w, n, shard * n, enc)
    if blob is not None and n > 8192:
        return native_columns(w, n, shard * n, blob)
    return w.columns(w.fields(n, start=shard * n), enc)


def cpu_port_rate(w, ft, enc, seconds=10.0, n=None, threads=None):
    """Decisions/s of the C port (oracle/c/check_ref.c) on all host cores over a bounded sample."""
    from oracle import cref
    import ctypes
    n = n or min(w.default_n, 1 << 20)
    threads = threads or (os.cpu_count() or 1)
    b = shard_columns(w, n, 0, enc, ft.blob)
    cols = [np.ascontiguousarray(c) for c in b.columns]
    ptrs = (ctypes.c_void_p * len(cols))(*[c.ctypes.data for c in cols])
    sizes = (ctypes.c_size_t * len(cols))(*[c.nbytes for c in cols])
    bb = cref._Batch(b.n, b.max_actions, NOW_NS, 0, ptrs, sizes, len(cols))
    out = np.zeros((b.n, b.max_actions), dtype=np.uint8)
    buf = ctypes.create_string_buffer(ft.blob, len(ft.blob))
    lib = cref.lib()
    lib.cref_check(buf, len(ft.blob), ctypes.byref(bb), out.ctypes.data, threads)  # warm
    t0 = time.perf_counter()
    passes = 0
    while True:
        rc = lib.cref_check(buf, len(ft.blob), ctypes.byref(bb), out.ctypes.data, threads)
        assert rc == 0
        passes += 1
        dt = time.perf_counter() - t0
        if dt >= seconds or passes >= 10000:
            break
    return passes * b.n * b.max_actions / dt, threads, passes, b.n, dt


def go_probe():
    """`go version` (the reference's own engine could only be timed with a Go >= 1.25 toolchain and its module cache)."""
    try:
        r = subprocess.run(["go", "version"], capture_output=True, text=True, timeout=10)
        return r.stdout.strip() or "go: no output"
    except (OSError, subprocess.SubprocessError):
        return "not found"


def run_go_reference(args, w):
    """The reference's own Go engine through baseline/go/engine_gpubaseline_test.go, when a Go toolchain and a cerbos
    checkout with its module cache are present (CERBOS_B200_REF_CHECKOUT or baseline/_ref/cerbos); None otherwise."""
    import shutil
    import tempfile
    if go_probe() == "not found":
        return None
    checkout = os.environ.get("CERBOS_B200_REF_CHECKOUT") or os.path.join(ROOT, "baseline", "_ref", "cerbos")
    if not os.path.isdir(os.path.join(checkout, "internal", "engine")):
        return None
    try:
        work = tempfile.mkdtemp(prefix="cerbos_b200_ref_")
        subprocess.run([sys.executable, os.path.join(ROOT, "tools", "export_workload.py"), "--workload", w.name, "--out", work, "--requests", str(1 << 20),
                        "--want"], check=True, capture_output=True, timeout=1200)
        shutil.copy(os.path.join(ROOT, "baseline", "go", "engine_gpubaseline_test.go"), os.path.join(checkout, "internal", "engine"))
        env = dict(os.environ, CERBOS_B200_WORKLOAD_DIR=work, CERBOS_B200_SECONDS=str(max(10.0, args.cpu_seconds)), GOFLAGS="-mod=mod")
        r = subprocess.run(["go", "test", "./internal/engine", "-run", "TestGPUBaseline", "-v", "-count=1"], cwd=checkout, env=env, capture_output=True,
                           text=True, timeout=1800)
        for ln in r.stdout.splitlines():
            if "GPU_BASELINE_RESULT " in ln:
                return json.loads(ln.split("GPU_BASELINE_RESULT ", 1)[1])
    except Exception as e:  # noqa: BLE001 -- any failure means "not available": the port is timed instead
        sys.stderr.write(f"go reference arm unavailable: {e}\n")
    return None


def run_reference(args):
    """--impl reference: the CPU path alone, rank 0 only."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    w = get_workload(args.workload)
    go = run_go_reference(args, w)
    if go is not None:
        print(json.dumps({
            "impl": "reference", "metric": METRIC, "value": go["value"], "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": None, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u64", "data": "synthetic",
            "config": {"workload": workload_label(w, args.gpus, args.requests or w.default_n), "go_toolchain": go.get("go"),
                       "note": "the reference's own engine.Check (baseline/go/engine_gpubaseline_test.go), GOMAXPROCS client goroutines, batches of 1024"},
            "cpu_baseline": {"value": go["value"], "unit": UNIT, "cores": go["cores"], "kind": "reference",
                             "sample": f"{go['inputs']} inputs of the workload stream for {go['seconds']:.1f} s"},
            "e2e": {"value": go["value"], "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))
        return
    import workloads as W
    _, ft, enc = W.build(w)
    # one "step" = a bounded sample: the first 2^20 requests of the workload's stream on all host threads
    n = min(w.default_n, 1 << 20)
    from oracle import cref
    import ctypes
    threads = os.cpu_count() or 1
    b = shard_columns(w, n, 0, enc, ft.blob)
    cols = [np.ascontiguousarray(c) for c in b.columns]
    ptrs = (ctypes.c_void_p * len(cols))(*[c.ctypes.data for c in cols])
    sizes = (ctypes.c_size_t * len(cols))(*[c.nbytes for c in cols])
    bb = cref._Batch(b.n, b.max_actions, NOW_NS, 0, ptrs, sizes, len(cols))
    out = np.zeros((b.n, b.max_actions), dtype=np.uint8)
    buf = ctypes.create_string_buffer(ft.blob, len(ft.blob))
    lib = cref.lib()
    for _ in range(args.warmup):
        lib.cref_check(buf, len(ft.blob), ctypes.byref(bb), out.ctypes.data, threads)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        rc = lib.cref_check(buf, len(ft.blob), ctypes.byref(bb), out.ctypes.data, threads)
        assert rc == 0
    dt = time.perf_counter() - t0
    value = args.steps * b.n * b.max_actions / dt
    sample = f"{b.n} requests x {b.max_actions} actions per step ({w.name} stream prefix), {threads} threads"
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "u64", "data": "synthetic",
        "config": {"workload": workload_label(w, args.gpus, args.requests or w.default_n), "sample_requests_per_step": b.n, "actions_per_request": b.max_actions,
                   "go_toolchain": go_probe(),
                   "note": "CPU port of the reference algorithm (oracle/c/check_ref.c) on all host threads, a 2^20-request prefix of the "
                           "workload's stream per step; the reference's own Go engine needs a Go toolchain + module cache "
                           "(baseline/go/ holds the harness source), absent from this image"},
        "cpu_baseline": {"value": value, "unit": UNIT, "cores": threads, "kind": "port", "sample": sample},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }))


def verify_images(w, blob, host_batches, images, kbytes):
    """Result images against the C port of the reference algorithm (oracle/): bit for bit over every request up to 2^24
    per batch, beyond that over a striped sample (every 16th run of 65 536 requests) as BASELINE.md 2.4 prescribes.
    -> (mismatching bytes, requests compared)"""
    from oracle import cref
    bad = cmp = 0
    for hb, img in zip(host_batches, images):
        n = hb.n
        if n <= (1 << 24):
            spans = [(0, n)]
        else:
            spans = [(s0, min(65536, n - s0)) for s0 in range(0, n, 16 * 65536)]
        for s0, cnt in spans:
            if (s0, cnt) == (0, n):
                cols = hb.columns
            else:   # a sub-batch: per-request columns sliced, batch-level tables as they are
                cols = list(hb.columns)
                cols[0] = np.ascontiguousarray(hb.columns[0][s0:s0 + cnt])
                cols[1] = np.ascontiguousarray(hb.columns[1][s0:s0 + cnt])
                cols[2] = np.ascontiguousarray(hb.columns[2][:, s0:s0 + cnt])
                cols[3] = np.ascontiguousarray(hb.columns[3][:, s0:s0 + cnt])
            want = cref.check(blob, cols, cnt, hb.max_actions, NOW_NS, 0, n_threads=os.cpu_count() or 1)
            want_bits = np.packbits((want == 1).astype(np.uint8), axis=1, bitorder="little")[:, :kbytes].reshape(-1)
            bad += int((img[s0 * kbytes:(s0 + cnt) * kbytes] != want_bits).sum())
            cmp += cnt
    return bad, cmp


def dump_decisions(out_dir, wname, images, n, K, kbytes, budget=48 << 20):
    """Writes <workload>_batch<j>_effects.npy (float32 [rows, K]: 1 ALLOW, 2 DENY) for every batch j in `images` and
    <workload>_rows.npy (float64: the request indices of those rows): a seeded sample of rows, the same on every run with
    the same request count, actions and batch set, at most `budget` bytes in all."""
    os.makedirs(out_dir, exist_ok=True)
    n_rows = max(1, min(n, budget // (4 * K * len(images) + 8)))
    rows = np.sort(np.random.default_rng(0x5EED).choice(n, size=n_rows, replace=False))
    np.save(os.path.join(out_dir, f"{wname}_rows.npy"), rows.astype(np.float64))
    for j, img in sorted(images.items()):
        bm = np.asarray(img).reshape(n, kbytes)[rows]
        bits = np.unpackbits(bm, axis=1, bitorder="little")[:, :K]
        np.save(os.path.join(out_dir, f"{wname}_batch{j}_effects.npy"), np.where(bits == 1, 1, 2).astype(np.float32))


def measure(args, ctx, w, blob, enc, table, dev, rank, world, local_rank, n, primary=True):
    """Times the device-resident path of one workload; returns the result fragment (see main)."""
    import torch
    import torch.distributed as dist
    from cerbos_b200.device import DeviceBatch
    from cerbos_b200.dist import all_gather_bitmaps

    K = len(w.actions)
    n_buf = 2 if n >= (1 << 22) else 4 if n >= (1 << 18) else 1
    batches, host_batches = [], []
    for j in range(n_buf):   # distinct batches: this rank's shard, n_buf consecutive windows of the workload stream
        hb = shard_columns(w, n, rank * n_buf + j, enc, blob)
        host_batches.append(hb)
        batches.append(DeviceBatch(hb, dev))
    footprint = sum(b.nbytes() for b in batches)
    l2_mb = getattr(torch.cuda.get_device_properties(dev), "L2_cache_size", 0) / 1e6
    kbytes = batches[0].kbytes
    calls = [b.prepare(table, NOW_NS) for b in batches]
    views = [b.bitmap[: n * kbytes] for b in batches]
    torch.cuda.synchronize()
    # Steps are independent batches.  Small batches (C2: a launch is ~20 us) are issued round-robin on two streams so that
    # the tail of one launch overlaps the head of the next; a C3-sized launch fills the GPU for milliseconds: one stream.
    n_streams = args.streams if args.streams else (2 if n < (1 << 22) else 1)
    n_streams = max(1, min(n_streams, n_buf))
    while n_buf % n_streams:
        n_streams -= 1
    streams = [torch.cuda.Stream() for _ in range(n_streams)]
    stream = streams[0]
    torch.cuda.set_stream(stream)
    stream_h = stream.cuda_stream
    stream_hs = [st.cuda_stream for st in streams]
    assert all(h != 0 for h in stream_hs) and torch.cuda.current_stream().cuda_stream == stream_h

    # Multi-GPU result exchange (primary workload only).  Default: every rank's results land in every rank's gather
    # buffer over NVLink peer memory (cerbos_b200.dist.PeerGather): small slices are stored by the check kernels
    # themselves, large ones are pushed by the copy engines behind the kernel; a flag release follows, no collective
    # kernel runs.  Fallback (CERBOS_B200_NCCL_GATHER=1, or CUDA IPC unavailable): asynchronous NCCL all-gather.
    gather_mode = "none"
    pg, gcalls = None, None
    n_gbuf = n_buf if n_buf >= 4 else 4     # gather buffers (a multiple of n_buf and of n_streams)
    if world > 1 and primary:
        ok = 0
        no_exchange = os.environ.get("CERBOS_B200_NO_GATHER") == "1"   # diagnosis only
        if os.environ.get("CERBOS_B200_NCCL_GATHER") != "1" and kbytes <= 8 and not no_exchange:
            try:
                from cerbos_b200.dist import PeerGather
                # more gather buffers than batches: a buffer is reused n_gbuf launches later, so a rank only ever waits for
                # what its peers finished n_gbuf - 1 launches ago (ranks drift apart by a few percent per launch)
                pg = PeerGather(ctx, n * kbytes, n_gbuf)
                gcalls = [table.prepared_gather_call(batches[i % n_buf].ptrs, batches[i % n_buf].sizes, batches[i % n_buf].n, batches[i % n_buf].max_actions,
                                                     pg.bufs[i], pg.lane_flags(i % n_streams), rank, n * kbytes, NOW_NS)
                          for i in range(n_gbuf)]
                ok = 1
            except Exception as e:  # noqa: BLE001 -- any failure here just selects the NCCL path on every rank
                sys.stderr.write(f"[rank {rank}] peer gather unavailable ({e}); using NCCL\n")
        t_ok = torch.tensor([ok], dtype=torch.int32, device=dev)
        dist.all_reduce(t_ok, op=dist.ReduceOp.MIN)
        gather_mode = "peer-memory" if int(t_ok.item()) == 1 else "nccl-all-gather"
        if gather_mode != "peer-memory":
            pg, gcalls = None, None
        if no_exchange:
            gather_mode = "none (diagnosis)"
        elif pg is None:       # NCCL orders its collective after torch's current stream only: one issuing stream
            n_streams, streams, stream_hs = 1, streams[:1], stream_hs[:1]
        elif n * kbytes >= (1 << 20):
            gather_mode = "peer-memory: copy engines push each rank's slice to every peer behind the kernel"
        else:
            gather_mode = "peer-memory: the check kernels store into every peer's buffer"
    gathered = [torch.empty(world * n * kbytes, dtype=torch.uint8, device=dev) for _ in range(n_buf)] if (world > 1 and primary and pg is None) else None
    pending = []
    it = [0]          # launches issued so far (warm-up included): numbers the gather steps

    def image(j):   # this rank's packed result bitmap of batch j (1 bit per decision, bit set = ALLOW)
        if pg is not None:
            return pg.read(j)[rank * n * kbytes:(rank + 1) * n * kbytes]
        return batches[j].bitmap[: n * kbytes].cpu().numpy()

    def launch():
        g = it[0]
        it[0] += 1
        j = g % n_buf
        lane = g % n_streams            # == j % n_streams: a buffer always travels on the same stream
        sh = stream_hs[lane]
        if pg is not None:
            # gather buffers rotate: launch g-(n_gbuf-1) must have landed on this rank before its stream moves on.  Launches
            # are numbered per stream ("lane"), so that every flag array only ever counts up.
            k = g - (n_gbuf - 1)
            if k >= 0:
                gcalls[g % n_gbuf](g // n_streams + 1, sh, k // n_streams + 1, pg.local_flags(k % n_streams))
            else:
                gcalls[g % n_gbuf](g // n_streams + 1, sh, 0, None)
            return
        calls[j](sh)
        if gathered is not None and gather_mode != "none (diagnosis)":
            if len(pending) >= n_buf - 1:          # buffers are reused after n_buf launches: retire the oldest gather
                pending.pop(0).wait()
            _, work = all_gather_bitmaps(views[j], gathered[j], async_op=True)
            pending.append(work)

    def drain():
        if pg is not None:
            for lane in range(n_streams):          # the last launch issued on every stream (a stream finishes in order)
                last = [g for g in range(max(0, it[0] - n_streams), it[0]) if g % n_streams == lane]
                if last:
                    pg.wait(last[-1] // n_streams + 1, stream_hs[lane], lane)
            return
        while pending:
            pending.pop(0).wait()

    def join_streams():
        for st in streams[1:]:
            e = torch.cuda.Event()
            e.record(st)
            stream.wait_event(e)

    def sync_all():
        drain()
        for h in stream_hs:
            ctx.sync(h)
        torch.cuda.synchronize()
        if world > 1 and primary:
            dist.barrier()

    # warm-up launches, then calibrate batches_per_step so that one step is >= ~10 ms of device work
    for _ in range(max(3, n_gbuf if pg is not None else n_buf)):
        launch()
    sync_all()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(n_buf * n_streams):
        launch()
    drain()
    join_streams()
    e1.record(stream)
    sync_all()
    t_launch_ms = e0.elapsed_time(e1) / (n_buf * n_streams)
    m = max(1, int(np.ceil(args.step_ms / max(t_launch_ms, 1e-4))))
    m = ((m + n_buf - 1) // n_buf) * n_buf if m > 1 else 1
    if world > 1 and primary:
        tm = torch.tensor([m], dtype=torch.int64, device=dev)
        dist.all_reduce(tm, op=dist.ReduceOp.MAX)
        m = int(tm.item())
    if args.batches_per_step:
        m = args.batches_per_step
    for _ in range(args.warmup):
        for _ in range(m):
            launch()
    sync_all()
    launches0 = ctx.launch_count()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(local_rank) as clocks:
        torch.cuda.synchronize()
        ev0.record(stream)
        for st in streams[1:]:
            st.wait_event(ev0)               # no stream starts before the start event
        t_host0 = time.perf_counter()
        for _ in range(args.steps * m):
            launch()
        host_issue_ms = (time.perf_counter() - t_host0) * 1e3 / (args.steps * m)   # host time to enqueue one batch
        drain()                              # the last exchanges are part of the timed work
        join_streams()
        ev1.record(stream)
        torch.cuda.synchronize()
    if world > 1 and primary:
        dist.barrier()
    total_ms = ev0.elapsed_time(ev1)
    launches = ctx.launch_count() - launches0
    for h in stream_hs:
        ctx.sync(h)
    if args.dump_outputs and primary and rank == 0:
        # the batches the last timed step evaluated (its m launches, numbered it[0] - m .. it[0] - 1, rotate over n_buf)
        dump_decisions(args.dump_outputs, w.name, {j: image(j) for j in {g % n_buf for g in range(it[0] - m, it[0])}}, n, K, kbytes)
    if world > 1 and primary:
        tmax = torch.tensor([total_ms], dtype=torch.float64, device=dev)
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        total_ms = float(tmax.item())
    per_step_ms = total_ms / args.steps
    wn = world if primary else 1
    value = wn * m * n * K / (per_step_ms * 1e-3)

    # kernel-only duration: (a) the whole device work of one call issued alone, (b) the dominant check kernel alone, from
    # the library's own CUDA events recorded on the launching stream around that kernel (cgpu_profile)
    step_ms = []
    p0, p1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ctx.profile(True)
    for i in range(min(args.steps * m, 30)):
        p0.record()
        calls[i % n_buf](stream_h)
        p1.record()
        p1.synchronize()
        step_ms.append(p0.elapsed_time(p1))
    k_sum, k_n = ctx.profile(False)
    kern_ms_mean = k_sum / max(k_n, 1)
    kcfg = ctx.last_kernel_config()
    peak, peak_src = load_peaks()
    algo_bytes = w.bytes_per_request() * n
    # The library's events bracket the first check kernel of a call.  When that kernel is not where the time goes (a table
    # whose requests are deferred to the general kernel behind it), the roofline is taken on the whole call instead.
    kernel_dominates = kern_ms_mean >= 0.5 * statistics.mean(step_ms)
    dominant_ms = kern_ms_mean if kernel_dominates else statistics.mean(step_ms)
    achieved = algo_bytes / (dominant_ms * 1e-3) / 1e9

    # correctness of what was timed: the result images the timed loop left behind, every rotating batch, against the oracle
    verified, compared = None, 0
    if not args.no_verify:
        for h in stream_hs:
            ctx.sync(h)
        torch.cuda.synchronize()
        images = [image(j) for j in range(n_buf)]
        bad, compared = verify_images(w, blob, host_batches, images, kbytes)
        if world > 1 and primary:
            tb = torch.tensor([bad], dtype=torch.int64, device=dev)
            dist.all_reduce(tb)
            bad = int(tb.item())
            if pg is not None and bad == 0:
                # every rank also holds every other rank's slice: compare the whole gathered image across ranks
                hsh = torch.tensor([int(np.frombuffer(pg.read(0).tobytes(), dtype=np.uint64).sum() & ((1 << 62) - 1))], dtype=torch.int64, device=dev)
                hs = [torch.zeros_like(hsh) for _ in range(world)]
                dist.all_gather(hs, hsh)
                bad = 0 if len({int(x.item()) for x in hs}) == 1 else -1
        verified = bad == 0
        if not verified:
            sys.stderr.write(f"[rank {rank}] VERIFY FAILED ({w.name}): {bad} result bytes differ from the oracle\n")

    res = {
        "value": value, "ms_per_step": per_step_ms, "batches_per_step": m, "requests_per_batch": n, "actions_per_request": K,
        "ms_per_batch": per_step_ms / m, "host_issue_ms_per_batch": host_issue_ms, "streams": n_streams, "gather_mode": gather_mode,
        "l2": f"rotating {n_buf} distinct batches, {footprint / 1e6:.0f} MB of columns; L2 {l2_mb:.0f} MB", "kernel": kcfg,
        "gpu_launches": int(launches),
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                     "peak_source": peak_src, "algorithmic_bytes_per_launch": algo_bytes,
                     "kernel": ("check_kernel<false,2> (general body draining the deferral list; timed as the whole call)" if not kernel_dominates else
                                ("cb_spec_uc" if kcfg.get("smem_bytes") else "cb_spec_uc_global") if kcfg.get("unique_conditions") and kcfg.get("table_specialised") else
                                "cb_spec_tiles" if kcfg.get("table_specialised") else "check_kernel"),
                     "kernel_ms_mean": kern_ms_mean,
                     "device_call_ms_mean": statistics.mean(step_ms), "device_call_ms_min": min(step_ms),
                     "call_achieved": algo_bytes / (statistics.mean(step_ms) * 1e-3) / 1e9,
                     "kernel_share_of_call": kern_ms_mean / statistics.mean(step_ms),
                     "note": "kernel_ms_mean: the dominant check kernel alone, CUDA events recorded by the library on the launching "
                             "stream around that kernel, one call at a time after the timed region; device_call_ms_*: events around "
                             "one whole cgpu_check_device call issued alone (pre-pass + check kernel + drain kernel)"},
        "clocks": clocks.summary(), "verified_vs_oracle": verified, "verified_requests": compared,
    }
    res["_host_batches"] = host_batches
    res["_kbytes"] = kbytes
    if pg is not None:
        torch.cuda.synchronize()
        dist.barrier()
        pg.close()
    del batches, calls, views
    torch.cuda.empty_cache()
    return res


def measure_e2e(args, table, hb, K, world, dev, n_slots):
    """End to end through the host-buffer C ABI on THIS rank's GPU / PCIe link: pinned host columns, H2D + kernels + D2H
    inside the timing.  Every rank runs it on its own shard; the aggregate is n_gpus x requests over the slowest rank.
    Headline: cgpu_check_narrow (the batch in its narrow wire form, widened on the device); cgpu_check on the canonical
    8-byte columns is timed beside it (`wide`)."""
    import torch
    import torch.distributed as dist
    from cerbos_b200 import narrow as NW

    def pin(a):
        a = np.ascontiguousarray(a)
        t = torch.empty(max(a.nbytes, 1), dtype=torch.uint8).pin_memory()
        t.numpy()[: a.nbytes] = a.view(np.uint8).reshape(-1)
        return t.data_ptr(), t

    def timed(fn):
        for _ in range(3):
            fn()
        if world > 1:
            dist.barrier()
        t0 = time.perf_counter()
        for _ in range(args.e2e_steps):
            fn()
        dt = (time.perf_counter() - t0) / args.e2e_steps
        if world > 1:
            td = torch.tensor([dt], dtype=torch.float64, device=dev)
            dist.all_reduce(td, op=dist.ReduceOp.MAX)
            dt = float(td.item())
        return dt

    pinned = [pin(c) for c in hb.columns]
    ptrs = [p for p, _ in pinned]
    sizes = [int(np.ascontiguousarray(c).nbytes) for c in hb.columns]
    out = torch.empty(hb.n * hb.max_actions, dtype=torch.uint8).pin_memory()
    dt_wide = timed(lambda: table.check_into(ptrs, sizes, hb.n, hb.max_actions, out.data_ptr(), NOW_NS, 0))
    wide = {"value": world * hb.n * K / dt_wide, "unit": UNIT, "h2d_bytes_per_step": int(sum(sizes)), "d2h_bytes_per_step": int(hb.n * hb.max_actions),
            "ms_per_step": dt_wide * 1e3, "call": "cgpu_check (canonical 8-byte columns)"}
    nb = NW.narrow_batch(hb, n_slots)
    if nb is None:
        res = dict(wide)
    else:
        out.zero_()
        b, nr, keep = table.prepare_narrow(nb, NOW_NS, 0, pin=pin)
        dt = timed(lambda: table.check_narrow_into(b, nr, out.data_ptr()))
        res = {"value": world * hb.n * K / dt, "unit": UNIT, "h2d_bytes_per_step": nb.wire_bytes(), "d2h_bytes_per_step": int(hb.n * hb.max_actions),
               "ms_per_step": dt * 1e3, "call": "cgpu_check_narrow (narrow wire form: 16-bit ids, u32 / f32 / u8 slot columns, 32-bit string heap; widened on the device)",
               "wire_bytes_per_request": nb.wire_bytes() / hb.n, "wide": wide}
    res.update({"n_gpus": world, "requests_per_step_per_gpu": hb.n,
                "note": "every rank calls it on its own shard over its own PCIe link: pinned host columns -> H2D (chunked, overlapped) -> kernels "
                        "-> D2H effect bytes (1 byte per decision); aggregate = n_gpus x requests / slowest rank"})
    return res, out


def measure_host_encode(w, blob, table, K, n=1 << 16):
    """The host stage a PDP adds in front of cgpu_check: serialized enginev1.CheckInput messages -> columns (native encoder,
    cgpu_encode, all host threads), alone and followed by cgpu_check -- reported separately from `e2e`, whose inputs are
    already encoded (SURVEY.md 7)."""
    import ctypes
    from cerbos_b200 import capi, wire
    inputs = w.inputs(w.fields(n), range(n))
    msgs = [wire.check_input(i) for i in inputs]
    keep = [ctypes.create_string_buffer(m, len(m)) for m in msgs]
    ptrs = (ctypes.c_void_p * n)(*[ctypes.addressof(b) for b in keep])
    lens = (ctypes.c_size_t * n)(*[len(m) for m in msgs])
    ne = capi.NativeEncoder(blob)
    eb = ne.encode_raw(ptrs, lens, n)
    col_bytes = sum(int(eb.batch().column_bytes[i]) for i in range(capi.N_COLUMNS))
    table.check_encoded(eb, NOW_NS)
    eb.free()
    reps = 5
    t0 = time.perf_counter()
    for _ in range(reps):
        eb = ne.encode_raw(ptrs, lens, n)
        eb.free()
    t_enc = (time.perf_counter() - t0) / reps
    t0 = time.perf_counter()
    for _ in range(reps):
        eb = ne.encode_raw(ptrs, lens, n)
        table.check_encoded(eb, NOW_NS)
        eb.free()
    t_both = (time.perf_counter() - t0) / reps
    # the same with the native narrowing pass in between: cgpu_encode -> cgpu_narrow_build -> cgpu_check_narrow (no Python on the path)
    narrow_path = None
    try:
        if os.environ.get("CERBOS_B200_BENCH_NATIVE_NARROW") != "1":
            # opt-in: cgpu_narrow_build's output is verified byte for byte against its specification on the CPU, but this leg
            # (its page-locked block handed to cgpu_check_narrow) has not run on a device yet -- not in the default bench line
            raise RuntimeError("skipped (set CERBOS_B200_BENCH_NATIVE_NARROW=1)")
        import numpy as _np
        out = None
        want = None
        t0 = time.perf_counter()
        for _ in range(reps):
            eb = ne.encode_raw(ptrs, lens, n)
            nz = eb.narrow(2)
            if nz is None:
                eb.free()
                raise RuntimeError("batch not narrowable")
            b, nr = nz.view(NOW_NS)
            if out is None or out.shape != (int(b.n_requests), max(int(b.max_actions), 1)):
                out = _np.empty((int(b.n_requests), max(int(b.max_actions), 1)), dtype=_np.uint8)   # the library writes n x max_actions bytes
            table.check_narrow_into(b, nr, out.ctypes.data)
            nz.free()
            eb.free()
        t_narrow = (time.perf_counter() - t0) / reps
        eb = ne.encode_raw(ptrs, lens, n)
        want = table.check_encoded(eb, NOW_NS)
        eb.free()
        narrow_path = {"decisions_per_s": n * K / t_narrow, "equals_canonical_call": bool((_np.asarray(want).reshape(out.shape) == out).all())}
    except Exception as e:  # noqa: BLE001 -- an optional extra line of the report, never the reason a bench run fails
        narrow_path = {"error": repr(e)[:200]}
    ne.close()
    threads = int(os.environ.get("CERBOS_B200_ENCODE_THREADS", "0")) or min(32, os.cpu_count() or 1)
    return {"requests_per_s": n / t_enc, "column_gb_per_s": col_bytes / t_enc / 1e9, "wire_bytes_per_request": sum(len(m) for m in msgs) / n,
            "threads": threads, "encode_plus_check_decisions_per_s": n * K / t_both, "encode_narrow_check": narrow_path,
            "sample": f"{n} serialized CheckInput messages of the workload per call (cgpu_encode, then cgpu_encode + cgpu_check, then "
                      "cgpu_encode + cgpu_narrow_build + cgpu_check_narrow)"}


WORKLOAD_DOC = {
    "C1": "C1: 1 resource policy, 3 actions, role-only rules, 1024 requests (BASELINE.json configs[0])",
    "C2": "C2: 10 resource policies x 8 actions, 2 derived roles with CEL on request.resource.attr, 2^20 requests (BASELINE.json configs[1])",
    "C3": "C3: 100 scoped resource policies (3-level scope chains), 20 CEL conditions incl. string / list operations, 2^24 requests (BASELINE.json configs[2])",
    "C5": "C5: 1000 policies, deep CEL (nested condition trees, maps, comprehensions, JWT claims), Zipf-skewed kinds, 2^23 requests per GPU = 64M on 8 GPUs (BASELINE.json configs[4])",
}


def workload_label(w, world, n):
    """config.workload: the same string on both arms (ours / --impl reference)"""
    name = WORKLOAD_DOC.get(w.name, w.name)
    if w.name == "C3" and world > 1:
        name = f"C4: the C3 table, {world} x 2^{int(np.log2(n))} requests sharded over {world} GPUs (BASELINE.json configs[3]); " + name
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workload", default="C3")
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--e2e-steps", type=int, default=5)
    ap.add_argument("--cpu-seconds", type=float, default=10.0)
    ap.add_argument("--requests", type=int, default=0, help="override requests per batch per GPU (profiling only)")
    ap.add_argument("--streams", type=int, default=0, help="CUDA streams the batches are issued on round-robin (0 = 2 for small batches, 1 for large)")
    ap.add_argument("--step-ms", type=float, default=10.0, help="a step is as many batches as make at least this much device work")
    ap.add_argument("--batches-per-step", type=int, default=0, help="override the calibrated number of batches per step")
    ap.add_argument("--no-verify", action="store_true", help="skip the post-run comparison of the result images with the oracle")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-secondary", action="store_true", help="skip the C2 ride-along measurement at N = 1")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write a seeded sample of the last step's decisions as .npy files to DIR")
    args = ap.parse_args()
    if args.warmup < 3:
        args.warmup = 3
    if args.impl == "reference":
        return run_reference(args)

    import torch
    import torch.distributed as dist
    from cerbos_b200 import capi
    import workloads as W

    # kernels the library compiles with NVRTC at table load are cached on disk: keep that cache out of the source tree
    # and out of the user's home unless the caller chose a directory
    if "CERBOS_B200_CACHE_DIR" not in os.environ:
        import atexit
        import shutil
        import tempfile
        cache = tempfile.mkdtemp(prefix="cerbos_b200_nvrtc_")
        atexit.register(shutil.rmtree, cache, True)
        os.environ["CERBOS_B200_CACHE_DIR"] = cache

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: cerbos_b200 has no CPU fallback")
    torch.cuda.set_device(local_rank)
    dev = f"cuda:{local_rank}"
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(dev))

    from cerbos_b200.dist import broadcast_blob
    from cerbos_b200.encode import Encoder, manifest_from_blob
    ctx = capi.Context(local_rank)

    def load(wname):
        w = get_workload(wname)
        blob = None
        if rank == 0:       # rank 0 flattens the policies; the blob is broadcast over NCCL (SURVEY.md 8(e))
            _, ft, _ = W.build(w)
            blob = ft.blob
        blob = broadcast_blob(blob, dev)
        enc = Encoder(manifest_from_blob(blob))
        table = ctx.load_table(blob)
        spec_ready, spec_note = table.wait_ready()   # table-specialised kernels (NVRTC, background thread) are in place
        return w, blob, enc, table, spec_ready, spec_note

    w, blob, enc, table, spec_ready, spec_note = load(args.workload)
    # requests per batch per GPU: BASELINE.json quotes C3 on one GPU (2^24; C4 = the same per GPU on 8) and C5 as 64M over
    # 8 GPUs = 2^23 per GPU
    n = args.requests or {"C5": 1 << 23}.get(w.name, w.default_n)
    K = len(w.actions)
    r = measure(args, ctx, w, blob, enc, table, dev, rank, world, local_rank, n, primary=True)
    host_batches = r.pop("_host_batches")
    r.pop("_kbytes")
    wl_name = workload_label(w, world, n)
    result = {
        "metric": METRIC, "value": r["value"], "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": r["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "u64", "data": "synthetic",
        "config": {"workload": wl_name, "batches_per_step": r["batches_per_step"], "requests_per_batch_per_gpu": n,
                   "requests_per_step_per_gpu": n * r["batches_per_step"], "actions_per_request": K,
                   "global_requests_per_step": world * n * r["batches_per_step"], "ms_per_batch": r["ms_per_batch"],
                   "host_issue_ms_per_batch": r["host_issue_ms_per_batch"],
                   "parallelism": f"dp{world} (requests sharded by index; NCCL table broadcast; result exchange: {r['gather_mode']})",
                   "streams": r["streams"], "l2": r["l2"], "kernel": r["kernel"],
                   "specialised_kernels": spec_note if not spec_ready else "compiled for this table at load (NVRTC)"},
        "gpu_launches": r["gpu_launches"], "roofline": r["roofline"], "clocks": r["clocks"],
        "verified_vs_oracle": r["verified_vs_oracle"], "verified_requests_per_gpu": r["verified_requests"],
    }

    if not args.no_e2e:
        e2e, out = measure_e2e(args, table, host_batches[0], K, world, dev, len(enc.slots))
        if not args.no_verify:   # the host-buffer path returns effect bytes: compare them too (first 2^20 requests)
            from oracle import cref
            hb = host_batches[0]
            cnt = min(hb.n, 1 << 20)
            cols = list(hb.columns)
            cols[0] = np.ascontiguousarray(hb.columns[0][:cnt]); cols[1] = np.ascontiguousarray(hb.columns[1][:cnt])
            cols[2] = np.ascontiguousarray(hb.columns[2][:, :cnt]); cols[3] = np.ascontiguousarray(hb.columns[3][:, :cnt])
            want = cref.check(blob, cols, cnt, hb.max_actions, NOW_NS, 0, n_threads=os.cpu_count() or 1)
            e2e["verified_vs_oracle"] = bool((out.numpy()[: cnt * hb.max_actions].reshape(cnt, hb.max_actions) == want).all())
        result["e2e"] = e2e
    del host_batches
    if rank == 0 and world == 1 and not args.no_e2e:
        result["host_encode"] = measure_host_encode(w, blob, table, K)
    if rank == 0 and world == 1 and not args.no_cpu:   # the CPU baseline is reported at N = 1 only
        _, ft0, enc0 = W.build(w)
        v, threads, passes, ns, dt = cpu_port_rate(w, ft0, enc0, seconds=args.cpu_seconds)
        result["cpu_baseline"] = {"value": v, "unit": UNIT, "cores": threads, "kind": "port",
                                  "sample": f"{passes} passes over {ns} requests x {K} actions ({dt:.1f} s) of the "
                                            f"same {w.name} stream, oracle/c/check_ref.c"}
    table.release()
    if world == 1 and not args.no_secondary and w.name != "C2":
        # configs[1] rides along: same measurement on workload C2 (device-resident path only)
        w2, blob2, enc2, table2, ready2, note2 = load("C2")
        r2 = measure(args, ctx, w2, blob2, enc2, table2, dev, rank, 1, local_rank, w2.default_n, primary=False)
        r2.pop("_host_batches"); r2.pop("_kbytes")
        result["secondary"] = {"workload": WORKLOAD_DOC["C2"], "metric": METRIC, "unit": UNIT, **r2}
        table2.release()
    if rank == 0:
        print(json.dumps(result))
    ctx.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
