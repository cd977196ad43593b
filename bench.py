#!/usr/bin/env python
"""bench.py — env-steps/sec of the batched Overcooked step engine on N H100s (BASELINE.json metric).

One bench "step" = one pass of the hot path over one batch of synthetic input = one full 400-transition horizon of
the workload's environments.  The headline workload is BASELINE.json configs[1] (cramped_room, 65 536 environments
per GPU, uniform random joint actions, 400 steps): 26 214 400 joint transitions per GPU per step.  Environments shard
by index across GPUs with no data-path collective (weak scaling: per-GPU work is fixed); NCCL carries the run seed and
the final counters.

  value          whole-job env-steps/s with the action trace already resident in HBM: one launch of the fused
                 T-step rollout kernel K5 per bench step (ovc_rollout through the C ABI)
  e2e            the same metric through the public host-buffer API (HostRolloutPipeline): actions start in pinned HOST
                 memory, dense reward / done arrays end in HOST memory, every byte copied (and expanded) inside the
                 timed region
  roofline       the dominant kernel (K5) against the measured HBM copy peak (MEASURED_PEAKS.json): algorithmic bytes =
                 what the fused kernel must stream, 32 B per env-step (8 B actions in, 24 B outputs) + 2*4*S/T for the
                 record; the kernel is instruction-issue / latency bound, so `issue_bound` is the governing figure
  roofline_k1    the per-transition kernel K1 (400 launches from one CUDA graph), SURVEY 8(d)'s 160 B accounting
  configs        short timed legs of the other BASELINE configs (3, 4, the 2^20-env target, 5), each with its own
                 roofline and a CPU replay of 256 sampled environments (`spot_check`)
  --dump-outputs DIR   after the timed steps, what the last timed step computed, as DIR/<name>.npy (a fixed, seeded
                 sample of the environments; float32, or float64 where an int32 value needs more than 24 bits)
  cpu_baseline   the C restatement of the reference's transition (oracle/, kind "port") on the usable host cores, and
                 `reference_python`: the reference's OWN Python OvercookedEnv.step loop timed on the same cores in the
                 same run (oracle/_ref copy, oracle/ref_python_bench.py)

--impl reference times the CPU restatement with all usable host threads on the same workload (median of several
bounded samples) and carries the same `reference_python` object.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CLASSIC5 = ["cramped_room", "asymmetric_advantages", "coordination_ring", "forced_coordination", "counter_circuit"]
WORKLOADS = {
    # name: (layouts, envs per GPU, horizon, what it is)
    "config2": (["cramped_room"], 65536, 400, "BASELINE configs[1]"),
    "config3": (CLASSIC5, 262144, 400, "BASELINE configs[2]: mixed batch of the 5 classic layouts, stored segmented"),
    "config4": (["asymmetric_advantages"], 131072, 400, "BASELINE configs[3]: 1 048 576 envs over 8 GPUs = 131 072 per GPU"),
    "target2e20": (["cramped_room"], 131072, 400, "north_star target: cramped_room at 2^20 envs over 8 GPUs = 131 072 per GPU"),
    # config 5: PPO-style self-play rollout (K2 encode -> torch CNN -> multinomial -> K1 step), 262 144 envs on 8 GPUs
    "config5": (["cramped_room"], 32768, 400, "BASELINE configs[4]: 262 144 envs over 8 GPUs = 32 768 per GPU, policy in the loop"),
}
METRIC = "env-steps/sec (joint transitions)"
_REAL_STDOUT = None


def emit(line):
    """The one JSON line of this run, on the process's original stdout."""
    data = (json.dumps(line) + "\n").encode()
    if _REAL_STDOUT is None:
        sys.stdout.write(data.decode())
        sys.stdout.flush()
    else:
        os.write(_REAL_STDOUT, data)


def workload_string(name, n_envs=None):
    """`config.workload` — the SAME string in the engine arm and the reference arm."""
    layouts, n, horizon, _ = WORKLOADS[name]
    return "%s: %s, %d envs/GPU, %d-step horizon with auto-reset, uniform random joint actions" % (
        name, "+".join(layouts), n_envs or n, horizon)


def load_tensor_peak():
    """(dense bf16 TFLOP/s, source): the driver-measured burst figure (a kernel timed alone), else the profiling recipe's fallback."""
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        if "bf16_tflops" in d:
            return float(d["bf16_tflops"]), "measured (MEASURED_PEAKS.json bf16_tflops, burst)"
    return 989.0, "data sheet (H100 SXM, 700 W: 989 TFLOP/s dense bf16), not measured"


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "data sheet (H100 SXM: 3.35 TB/s HBM3), not measured"


# ---------------------------------------------------------------------------------------------------------------
# host cores: what this process may really use, and this rank's share of its GPU's NUMA node
# ---------------------------------------------------------------------------------------------------------------
def _parse_cpulist(s):
    out = []
    for part in s.strip().split(","):
        if not part:
            continue
        a, _, b = part.partition("-")
        out.extend(range(int(a), int(b or a) + 1))
    return out


def usable_cpus():
    cpus = sorted(os.sched_getaffinity(0))
    lim = 0
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            lim = -(-int(q) // int(p))
    except Exception:
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            p = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0 and p > 0:
                lim = -(-q // p)
        except Exception:
            pass
    return cpus[:lim] if 0 < lim < len(cpus) else cpus


def gpu_numa_node(index):
    """NUMA node of CUDA device `index` from sysfs (None if the platform does not say)."""
    try:
        import torch

        p = torch.cuda.get_device_properties(index)
        bdf = "%04x:%02x:%02x.0" % (p.pci_domain_id, p.pci_bus_id, p.pci_device_id)
        node = int(open("/sys/bus/pci/devices/%s/numa_node" % bdf).read())
        return node if node >= 0 else None
    except Exception:
        return None


def bind_rank_to_numa_share(local, world):
    """Pin this process (and every thread it creates afterwards: the expansion pool, the pinned-buffer first touch)
    to its share of the host: the usable CPUs of its GPU's NUMA node, divided by physical core among the ranks whose
    GPUs sit on the same node.  Returns a description for the bench line."""
    cpus = usable_cpus()
    info = {"usable_cpus": len(cpus), "numa_node": None, "bound_cpus": len(cpus), "ranks_sharing_node": world,
            "_original_affinity": sorted(os.sched_getaffinity(0))}
    try:
        # every rank's candidate CPUs: the usable CPUs of its GPU's NUMA node, or all usable CPUs where the lease has none there;
        # ranks with the SAME candidates share them (by physical core) — 8 ranks on a whole box get 16 CPUs each, two ranks
        # of a small lease whose CPUs all sit on one node get half of it each
        def candidates(g):
            nd = gpu_numa_node(g)
            if nd is not None:
                on_node = set(_parse_cpulist(open("/sys/devices/system/node/node%d/cpulist" % nd).read()))
                loc = [c for c in cpus if c in on_node]
                if loc:
                    return nd, tuple(loc)
            return None, tuple(cpus)

        cands = [candidates(g) for g in range(world)]
        node, mine = cands[local] if local < world else candidates(local)
        mine = list(mine)
        sharing = [g for g in range(world) if cands[g][1] == tuple(mine)] or [local]
        info["numa_node"] = node
        if len(sharing) > 1 and local in sharing:
            cores = {}
            for c in mine:  # group hardware threads by physical core
                try:
                    sib = min(_parse_cpulist(open("/sys/devices/system/cpu/cpu%d/topology/thread_siblings_list" % c).read()))
                except Exception:
                    sib = c
                cores.setdefault(sib, []).append(c)
            keys = sorted(cores)
            k, n = sharing.index(local), len(sharing)
            part = keys[len(keys) * k // n: len(keys) * (k + 1) // n]
            if part:
                mine = sorted(c for key in part for c in cores[key])
        os.sched_setaffinity(0, set(mine))
        info["bound_cpus"], info["ranks_sharing_node"] = len(mine), len(sharing)
        if info["numa_node"] is not None:  # and prefer that node's memory for what is allocated from here on (pinned buffers)
            try:
                import ctypes
                mask = ctypes.c_ulong(1 << info["numa_node"])
                rc = ctypes.CDLL(None, use_errno=True).syscall(238, 1, ctypes.byref(mask), 65)  # set_mempolicy(MPOL_PREFERRED)
                info["mempolicy"] = "preferred node %d" % info["numa_node"] if rc == 0 else "set_mempolicy failed (errno %d)" % ctypes.get_errno()
            except Exception as e:
                info["mempolicy"] = "unavailable: %r" % (e,)
    except Exception as e:  # never let placement break the measurement
        info["error"] = repr(e)[:120]
    return info


class ClockSampler(object):
    """nvidia-smi clock / throttle sampling DURING the timed region."""

    Q = "index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown," \
        "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, gpu_index):
        self.gpu, self.proc, self.path = gpu_index, None, None

    def start(self):
        try:
            fd, self.path = tempfile.mkstemp(suffix=".csv")
            os.close(fd)
            self.proc = subprocess.Popen(
                ["nvidia-smi", "-i", str(self.gpu), "--query-gpu=" + self.Q, "--format=csv,noheader,nounits", "-lms", "10"],
                stdout=open(self.path, "w"), stderr=subprocess.DEVNULL)
            time.sleep(0.3)  # let the sampler come up before the timed region starts
        except Exception:
            self.proc = None

    def stop(self):
        out = {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        if self.proc is None:
            return out
        time.sleep(0.05)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        try:
            for line in open(self.path):
                f = [x.strip() for x in line.split(",")]
                if len(f) < 9:
                    continue
                try:
                    sm.append(float(f[1])), mx.append(float(f[2]))
                except ValueError:
                    continue
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
            os.unlink(self.path)
        except Exception:
            pass
        if sm:
            # "under load" = samples at or above the median of the upper half (idle samples before / after drop out)
            hi = sorted(sm)[len(sm) // 2:]
            out.update(sm_mhz=float(np.median(hi)), sm_max_mhz=float(max(mx)), reasons=sorted(reasons), samples=len(sm))
        return out


# ---------------------------------------------------------------------------------------------------------------
# CPU arm: the oracle port on the usable host cores + the reference's own Python loop
# ---------------------------------------------------------------------------------------------------------------
def oracle_tables(layout_names, n_envs):
    from overcooked_ai_b200 import layout as L

    layouts = [L.compile_layout(n) for n in layout_names]
    tab, starts, S = L.build_tables(layouts)
    bounds = [n_envs * i // len(layouts) for i in range(len(layouts) + 1)]
    state = np.concatenate([np.repeat(starts[i:i + 1], bounds[i + 1] - bounds[i], 0) for i in range(len(layouts))])
    return tab, starts, S, np.ascontiguousarray(state)


class CpuSampler(object):
    """Bounded CPU samples of a workload through the oracle: tables, action trace and output pages are prepared once
    (untimed); every sample restarts from the standard start states and times the transitions only."""

    def __init__(self, layout_names, n_envs, T, horizon, threads):
        from oracle import cpu as oracle_cpu

        self.o, self.threads, self.n_envs, self.T, self.horizon = oracle_cpu, threads, n_envs, T, horizon
        self.tab, self.starts, self.S, self.state0 = oracle_tables(layout_names, n_envs)
        self.acts = np.random.RandomState(0).randint(0, 6, size=(T, n_envs, 2)).astype(np.int32)
        self.out = oracle_cpu.alloc_rollout_out(T, n_envs)
        self.state = self.state0.copy()

    def sample(self):
        np.copyto(self.state, self.state0)
        t0 = time.perf_counter()
        self.o.rollout(self.tab, self.starts, self.state, self.acts, horizon=self.horizon, flags=1, n_threads=self.threads, out=self.out)
        return self.n_envs * self.T / (time.perf_counter() - t0)


def cpu_port_samples(layout_names, horizon, n_samples, budget_s):
    """(values, description): >= 5 samples unless the budget runs out; thread count = what the process may use."""
    from oracle import cpu as oracle_cpu

    threads = oracle_cpu.max_threads()
    n_envs = 16384 if threads >= 16 else 4096
    T = horizon
    s = CpuSampler(layout_names, n_envs, T, horizon, threads)
    s.sample()  # warm: threads created once, pages touched
    vals, t0 = [], time.perf_counter()
    while len(vals) < n_samples and (len(vals) < 5 or time.perf_counter() - t0 < budget_s):
        vals.append(s.sample())
    return vals, threads, "%d samples x (%d envs x %d transitions) of %s through oracle/ovc_oracle.c, %d pinned threads " \
                          "(affinity mask / cgroup quota of this process), transitions only" % (len(vals), n_envs, T, "+".join(layout_names), threads)


def spread(vals):
    v = sorted(vals)
    return {"median": float(np.median(v)), "min": float(v[0]), "max": float(v[-1]), "n": len(v),
            "rel_spread": float((v[-1] - v[0]) / np.median(v)) if v else None}


def reference_python(layout="cramped_room", seconds=3.0):
    """The reference's own Python step on this machine's cores, in its own process (no CUDA context is forked)."""
    try:
        r = subprocess.run([sys.executable, os.path.join(ROOT, "oracle", "ref_python_bench.py"), "--layout", layout, "--seconds", str(seconds)],
                           capture_output=True, text=True, timeout=180)
        if r.returncode != 0:
            return {"unavailable": (r.stderr.strip().splitlines() or ["failed"])[-1][:200]}
        return json.loads(r.stdout.strip().splitlines()[-1])
    except Exception as e:
        return {"unavailable": repr(e)[:200]}


def cpu_baseline(layout_names, horizon, with_reference=True):
    vals, threads, what = cpu_port_samples(layout_names, horizon, n_samples=7, budget_s=10.0)
    out = {"value": float(np.median(vals)), "unit": "env-steps/s", "cores": threads, "cores_effective": threads, "kind": "port",
           "sample": what, "samples": spread(vals), "logical_cpus_online": os.cpu_count()}
    if with_reference:
        out["reference_python"] = reference_python(layout_names[0])
    return out


def run_reference(args, rank, world):
    """--impl reference: the CPU restatement on all usable host threads, same workload string, bounded samples."""
    if rank != 0:
        return
    layouts, n_envs, horizon, _ = WORKLOADS[args.workload]
    from oracle import cpu as oracle_cpu

    threads = oracle_cpu.max_threads()
    sample_envs = 16384 if threads >= 16 else 4096
    s = CpuSampler(layouts, sample_envs, horizon, horizon, threads)
    for _ in range(max(1, args.warmup)):
        s.sample()
    vals = [s.sample() for _ in range(max(5, args.steps))]
    value = float(np.median(vals))
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": "env-steps/s", "n_gpus": args.gpus,
        "steps": len(vals), "warmup": max(1, args.warmup), "ms_per_step": 1e3 * sample_envs * horizon / value, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "int32", "data": "synthetic",
        "config": {"workload": workload_string(args.workload), "state_words": s.S,
                   "bounded_sample": "each step = %d envs x %d transitions of that workload on the CPU; value = median over steps" % (sample_envs, horizon)},
        "cpu_baseline": {"value": value, "unit": "env-steps/s", "cores": threads, "cores_effective": threads, "kind": "port",
                         "sample": "%d steps x %d envs x %d transitions, oracle/ovc_oracle.c, %d pinned threads (affinity mask / cgroup quota)"
                                   % (len(vals), sample_envs, horizon, threads),
                         "samples": spread(vals), "logical_cpus_online": os.cpu_count(),
                         "reference_python": reference_python(layouts[0])},
        "e2e": {"value": value, "unit": "env-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    emit(line)


# ---------------------------------------------------------------------------------------------------------------
# engine legs
# ---------------------------------------------------------------------------------------------------------------
DUMP_ENVS = 2048  # environments sampled per rank for --dump-outputs: 40 MB for the headline workload


def dump_outputs(directory, n_envs, dev, rank, per_env=None, per_step=None):
    """Write DIR/<name>.npy for every array of `per_env` ([N, ...]) and `per_step` ([T, N, ...]), restricted to the same seeded
    sample of DUMP_ENVS environments in every run.  Integer values go out as float64 (event masks use 29 bits), the rest as
    float32; rank r > 0 writes <name>.rank<r>.npy."""
    import torch

    ids = torch.from_numpy(np.sort(np.random.RandomState(20261015).choice(n_envs, size=min(DUMP_ENVS, n_envs), replace=False))).to(dev)
    os.makedirs(directory, exist_ok=True)
    arrays = [(name, a, 0) for name, a in (per_env or {}).items()] + [(name, a, 1) for name, a in (per_step or {}).items()]
    for name, a, env_axis in arrays:
        x = a.index_select(env_axis, ids).cpu().numpy()
        x = x.astype(np.float64 if x.dtype in (np.int32, np.int64) else np.float32)
        np.save(os.path.join(directory, name + (".rank%d" % rank if rank else "") + ".npy"), x)
    np.save(os.path.join(directory, "env_ids" + (".rank%d" % rank if rank else "") + ".npy"), ids.cpu().numpy().astype(np.float64))


def fused_roofline(S, T, n_envs, launch_s, peak, peak_src):
    """Roofline object of one K5 launch (T transitions of n_envs environments)."""
    bytes_per = 32.0 + 2.0 * 4.0 * S / T
    achieved = n_envs * T * bytes_per / launch_s / 1e9
    r = {
        "bound": "hbm", "governing": "instruction issue / latency: the fused kernel streams 32 B per env-step and keeps the record on chip",
        "kernel": "ovc::rollout_kernel<S=%d> K5: T=%d transitions fused in one launch" % (S, T),
        "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak, "peak_source": peak_src,
        "algorithmic_bytes_per_env_step": bytes_per, "env_steps_per_launch": n_envs * T, "avg_launch_us": launch_s * 1e6,
        "note": "algorithmic bytes = 8 B actions in + 24 B outputs per env-step + the record once in and out per launch (2*4*S/T); "
                "launch duration = CUDA-event time of the timed region / launches",
    }
    return r


def spot_check_rollout(env, actions, out, n_samples=256, seed=1234):
    """SURVEY 8(d): replay `n_samples` sampled environments of the LAST pass on the CPU oracle and compare every
    output of every transition and the final records.  The pass must have started from the start states."""
    import torch

    from oracle import cpu as oracle_cpu

    N, T = env.n_envs, actions.shape[0]
    ids = np.sort(np.random.RandomState(seed).choice(N, size=min(n_samples, N), replace=False))
    tid = torch.from_numpy(ids).to(env.device)
    lay = env.env_layout_host[ids]
    state = np.ascontiguousarray(env._starts_host[lay])
    acts = np.ascontiguousarray(actions[:, tid].cpu().numpy().astype(np.int32))
    want = oracle_cpu.rollout(env._tab_host, env._starts_host, state, acts, horizon=env.horizon, flags=1, n_threads=1)
    bad = []
    for name, got, w in zip(("sparse", "shaped", "done", "events"), out, want):
        if not np.array_equal(got[:, tid].cpu().numpy(), w):
            bad.append(name)
    if not np.array_equal(env.state[tid].cpu().numpy(), state):
        bad.append("state")
    return ("ok" if not bad else "MISMATCH in " + ",".join(bad)), len(ids)


def engine_leg(name, dev, rank, world, seed, steps, warmup, peak, peak_src, clocks=None, envs=0, io=0, pdl=True, sampler=None, dump=None):
    """One workload: device-resident action trace, `steps` launches of K5, CUDA events, max over ranks; then the
    sampled CPU replay.  Returns (dict for the bench line, env, actions, out) — the caller may reuse the buffers.
    dump: a directory that receives the last timed launch's outputs (dump_outputs)."""
    import torch

    from overcooked_ai_b200 import dist as D
    from overcooked_ai_b200.batched import BatchedOvercookedEnv

    layouts, n_envs, horizon, what = WORKLOADS[name]
    n_envs = envs or n_envs
    T = horizon
    env = BatchedOvercookedEnv(layouts, n_envs, horizon=horizon, device=dev, auto_reset=True, io=io, pdl=pdl)
    S = env.state_words
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed + rank)
    actions = torch.randint(0, 6, (T, n_envs, 2), dtype=torch.int32, device=dev, generator=gen)
    out = env.alloc_rollout_out(T)
    env.reset()
    for _ in range(warmup):
        env.rollout(actions, out=out)
    D.barrier()
    torch.cuda.synchronize(dev)
    if sampler is not None:
        sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        env.rollout(actions, out=out)
    e1.record()
    torch.cuda.synchronize(dev)
    D.barrier()
    ms = e0.elapsed_time(e1)
    if dump is not None:
        dump_outputs(dump, n_envs, dev, rank, per_env={"state": env.state},
                     per_step={"sparse": out[0], "shaped": out[1], "done": out[2], "events": out[3]})
    if sampler is not None:
        # the timed region lasts a few milliseconds, less than one nvidia-smi sampling period: keep the SAME launches going
        # (untimed) for ~0.4 s so that the clock / throttle record really is taken under this load
        n_more = max(10, int(400.0 / max(ms / steps, 1e-3)))
        for _ in range(n_more):
            env.rollout(actions, out=out)
        torch.cuda.synchronize(dev)
        clocks = sampler.stop()
        clocks["sampled_over"] = "the timed region and %d more launches of the same kernel (~0.4 s, untimed)" % n_more
    steps_local = float(n_envs) * T * steps
    tot_steps, max_ms, tot_reward = D.reduce_counters(steps_local, ms, float(out[0].sum().item()), device=dev)
    env.reset()
    env.rollout(actions, out=out)
    torch.cuda.synchronize(dev)
    spot, n_spot = spot_check_rollout(env, actions, out)
    ok_all, _, _ = D.reduce_counters(1.0 if spot == "ok" else 0.0, 0, 0, device=dev)
    leg = {
        "workload": workload_string(name, n_envs), "what": what, "value": tot_steps / (max_ms * 1e-3), "unit": "env-steps/s",
        "steps": steps, "ms_per_step": max_ms / steps, "state_words": S, "gpu_launches": steps,
        "roofline": fused_roofline(S, T, n_envs, max_ms * 1e-3 / steps, peak, peak_src),
        "spot_check": spot if ok_all == world else "MISMATCH on some rank", "spot_check_envs_per_rank": n_spot,
        "sparse_reward_sum": tot_reward,
    }
    return leg, env, actions, out, clocks


def policy_leg(dev, rank, world, seed, steps, warmup, envs=0, dump=None):
    """BASELINE config 5: step + lossless_state_encoding feeding a random-init torch CNN policy (one CUDA graph per
    transition).  Spot check: an eager stretch whose sampled actions are recorded and replayed on the CPU oracle."""
    import torch

    from oracle import cpu as oracle_cpu
    from overcooked_ai_b200 import dist as D
    from overcooked_ai_b200.batched import BatchedOvercookedEnv
    from overcooked_ai_b200.selfplay import SelfPlayRollout

    layouts, n_envs, horizon, what = WORKLOADS["config5"]
    n_envs = envs or n_envs
    T = horizon
    torch.manual_seed(seed + rank)
    torch.backends.cudnn.benchmark = True
    env = BatchedOvercookedEnv(layouts, n_envs, horizon=horizon, device=dev, auto_reset=True)
    sp = SelfPlayRollout(env, use_graph=True)

    def timed(fn, k, w):
        for _ in range(w):
            fn(T // 4)
        D.barrier()
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(k):
            fn(T)
        e1.record()
        torch.cuda.synchronize(dev)
        D.barrier()
        return e0.elapsed_time(e1)

    ms = timed(sp.run, steps, warmup)
    if dump is not None:
        dump_outputs(dump, n_envs, dev, rank, per_env={"state": env.state, "actions": sp.actions, "values": sp.values,
                                                       "ret_sparse": sp.ret_sparse, "ret_mixed": sp.ret_mixed})
    ms_env = timed(sp.env_only, 2, 1) / 2
    tot_steps, max_ms, tot_reward = D.reduce_counters(float(n_envs) * T * steps, ms, float(sp.ret_sparse.sum().item()), device=dev)
    _, max_ms_env, _ = D.reduce_counters(0, ms_env, 0, device=dev)
    # ---- spot check: 60 eager transitions from a reset, actions of 256 sampled envs recorded, CPU replay ----
    env.reset()
    ids = np.sort(np.random.RandomState(7).choice(n_envs, size=min(256, n_envs), replace=False))
    tid = torch.from_numpy(ids).to(dev)
    rec_a, rec_o = [], []
    for _ in range(60):
        sp._transition()
        rec_a.append(sp.actions[tid].clone())
        rec_o.append([x[tid].clone() for x in (env.sparse, env.shaped, env.done, env.events)])
    torch.cuda.synchronize(dev)
    state = np.ascontiguousarray(env._starts_host[env.env_layout_host[ids]])
    acts = np.stack([a.cpu().numpy() for a in rec_a]).astype(np.int32)
    want = oracle_cpu.rollout(env._tab_host, env._starts_host, state, acts, horizon=horizon, flags=1, n_threads=1)
    bad = [nm for k, nm in enumerate(("sparse", "shaped", "done", "events"))
           if not np.array_equal(np.stack([o[k].cpu().numpy() for o in rec_o]), want[k])]
    if not np.array_equal(env.state[tid].cpu().numpy(), state):
        bad.append("state")
    ok_all, _, _ = D.reduce_counters(0.0 if bad else 1.0, 0, 0, device=dev)
    S = env.state_words
    l = env.layouts[0]
    # ---- the policy-side kernels on their own (CUDA events, on the states / activations the run left behind) ----
    kernels = {}
    if sp.fused_first_layer and sp.fused_wide and sp.fused_tail:
        from overcooked_ai_b200 import _native as NV

        def kernel_us(fn, reps=20):
            for _ in range(3):
                fn()
            torch.cuda.synchronize(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            torch.cuda.synchronize(dev)
            return e0.elapsed_time(e1) / reps * 1e3

        rows = 2 * n_envs
        w1, b1, w2, b2 = sp._wide
        t1, c1, th, ch, to, co = sp._tail
        k7 = kernel_us(lambda: env.encoded_linear(sp._wt0, sp._b0, out=sp._act0, neg_slope=0.2))
        k9 = kernel_us(lambda: NV.check(NV.lib().ovc_wide_layers(sp._act0.data_ptr(), rows, 512, w1.data_ptr(), b1.data_ptr(), 512, w2.data_ptr(),
                                                                 b2.data_ptr(), 160, 0.2, sp._z.data_ptr(), env._stream())))
        k8 = kernel_us(lambda: NV.check(NV.lib().ovc_policy_tail(sp._z.data_ptr(), rows, 160, 0.2, t1.data_ptr(), c1.data_ptr(), th.data_ptr(), ch.data_ptr(),
                                                                 th.shape[0], to.data_ptr(), co.data_ptr(), 0.3, 6, 1, sp._draw_counter.data_ptr(),
                                                                 sp.actions.data_ptr(), sp.values.data_ptr(), 0, env._stream())))
        flops = rows * 2.0 * (512 * 512 + 512 * 160)
        peak_tf, peak_src = load_tensor_peak()
        kernels = {"k7_encode_linear_us": k7, "k9_wide_layers_us": k9, "k8_policy_tail_us": k8,
                   "roofline_k9": {"bound": "tensor", "kernel": "ovc::wide_layers_kernel (wgmma, accumulators in registers): 512 -> 512 -> 160 for %d rows" % rows,
                                   "achieved": flops / (k9 * 1e-6) / 1e12, "peak": peak_tf, "unit": "TFLOP/s", "frac": flops / (k9 * 1e-6) / 1e12 / peak_tf,
                                   "peak_source": peak_src, "flops_per_launch": flops, "avg_launch_us": k9,
                                   "note": "timed alone, back to back (burst peak); achieved = 2 * rows * (512*512 + 512*160) / duration"}}
    return {
        "workload": "config5: %s, %d envs/GPU, self-play: %s -> policy (RllibPPOModel-shaped CNN, random init, shared; "
                    "every convolution folded into one matrix, selfplay.DenseGridPolicy; the two wide layers: %s) -> %s -> K1 step "
                    "-> returns (ovc_accumulate_returns), whole transition in one CUDA graph" % ("+".join(layouts), n_envs,
                    "K7 (lossless encoding + first layer + leaky ReLU from the packed records, observation never materialised)"
                    if sp.fused_first_layer else "K2 lossless encode bf16",
                    "K9, one wgmma kernel" if sp.fused_wide else "library GEMMs",
                    "K8 (the dense layers of 64, the heads and the Gumbel-max action draw in one kernel)" if sp.fused_tail else "Gumbel-max sampling"),
        "what": what, "value": tot_steps / (max_ms * 1e-3), "unit": "env-steps/s", "steps": steps, "ms_per_step": max_ms / steps,
        "dtype": "int32 env / bf16 activations / bf16 policy",
        # kernels of this library per transition: K7 (or K2), K9, K8 (or the draw kernel), K1, the return kernel
        "gpu_launches": (1 + int(sp.fused_wide) + int(sp.native_glue) + 1 + int(sp.native_glue)) * T * steps,
        "env_only": {"kernels": "K7 (encoding + first policy layer) + K1" if sp.fused_first_layer else "K2 + K1", "ms_per_400_transitions": max_ms_env, "env_steps_per_s_per_gpu": n_envs * T / (max_ms_env * 1e-3),
                     "share_of_pipeline_time": max_ms_env / (max_ms / steps),
                     "algorithmic_bytes_per_env_step": 2 * 4 * S + 32 + 4 * S + (2 * sp._act0.shape[1] * 2 if sp.fused_first_layer else
                                                                                  2 * l.width * l.height * 26 * sp.obs.element_size())},
        "spot_check": ("ok" if not bad else "MISMATCH in " + ",".join(bad)) if ok_all == world else "MISMATCH on some rank",
        "spot_check_envs_per_rank": len(ids), "sparse_reward_sum": tot_reward, "policy_kernels": kernels,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="config2", choices=sorted(WORKLOADS))
    ap.add_argument("--io", type=int, default=0, help="record I/O strategy of K1 (0 default, 1 TMA tensor, 2 TMA bulk, 3 direct)")
    ap.add_argument("--envs", type=int, default=0, help="override environments per GPU of the headline workload")
    ap.add_argument("--no-cpu", action="store_true", help="skip the cpu_baseline leg")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-configs", action="store_true", help="skip the short legs of the other BASELINE configs")
    ap.add_argument("--no-pdl", action="store_true", help="disable programmatic dependent launch between K1 launches")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed step's outputs (a seeded sample of the environments) "
                                                          "as DIR/<name>.npy, to compare two builds output for output")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == "b200" else args.warmup

    # stdout must carry exactly one JSON line, but NCCL printf()s its version banner to fd 1 at communicator
    # creation: park the real stdout, point fd 1 at stderr for the run, emit the JSON line on the real one.
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.dup(1)
    os.dup2(2, 1)
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    if args.impl == "reference":
        run_reference(args, rank, world)
        return

    import torch

    from overcooked_ai_b200 import dist as D
    from overcooked_ai_b200.batched import HostRolloutPipeline

    assert torch.cuda.is_available(), "bench.py needs a CUDA device (no CPU fallback)"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    host = bind_rank_to_numa_share(local, world)  # before any pinned allocation / worker thread exists
    host_affinity = host.pop("_original_affinity")
    D.init("nccl")
    seed = D.broadcast_seed(20260922, device=dev)
    peak, peak_src = load_peaks()

    if args.workload == "config5":
        leg = policy_leg(dev, rank, world, seed, args.steps, args.warmup, args.envs, dump=args.dump_outputs)
        if rank == 0:
            emit({"metric": METRIC, "value": leg["value"], "unit": "env-steps/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
                  "ms_per_step": leg["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                  "dtype": leg["dtype"], "data": "synthetic", "config": {"workload": leg["workload"], "parallelism": "env-index sharding x%d" % world},
                  "gpu_launches": leg["gpu_launches"], "env_only": leg["env_only"], "spot_check": leg["spot_check"]})
        return

    # ---- headline: the fused rollout kernel on the chosen workload; clocks sampled over exactly this region ----
    sampler = ClockSampler(local) if rank == 0 else None
    head, env, actions, out, clocks = engine_leg(args.workload, dev, rank, world, seed, args.steps, args.warmup, peak, peak_src,
                                                 envs=args.envs, io=args.io, pdl=not args.no_pdl, sampler=sampler, dump=args.dump_outputs)
    layouts, _, horizon, _ = WORKLOADS[args.workload]
    n_envs, T, S = env.n_envs, horizon, env.state_words

    # ---- the per-transition kernel K1 (400 launches from one CUDA graph), measured in the same run ----
    out_t = [tuple(o[t] for o in out) for t in range(T)]

    def pass_step():
        for t in range(T):
            env.step(actions[t], out=out_t[t])

    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        pass_step()
    torch.cuda.current_stream(dev).wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        pass_step()
    env.reset()
    for _ in range(3):
        graph.replay()
    D.barrier()
    torch.cuda.synchronize(dev)
    k1_steps = max(2, min(args.steps, 5))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(k1_steps):
        graph.replay()
    e1.record()
    torch.cuda.synchronize(dev)
    D.barrier()
    _, k1_ms, _ = D.reduce_counters(0, e0.elapsed_time(e1), 0, device=dev)
    del graph

    # ---- e2e: the same workload through the public host-buffer API ----
    def run_e2e(fmt, expand=False):
        """One HostRolloutPipeline format.  expand: rebuild the dense sparse / shaped / done arrays on this rank's host
        cores inside the timed region (the payload a host consumer indexes)."""
        narrow = fmt != "int32"
        codes = fmt in ("codes", "stream")
        stream = fmt == "stream"
        chunk = int(os.environ.get("OVC_E2E_CHUNK", "100" if stream else "200" if codes else "50"))
        pipe = HostRolloutPipeline(env, T, chunk=chunk, narrow=narrow, packed=fmt == "packed", codes=codes, stream=stream, host_buffers=2)
        if codes:
            from overcooked_ai_b200 import wire
            h_actions = torch.from_numpy(wire.pack_actions(actions.cpu().numpy())).pin_memory()
            dense = {"sparse": torch.empty((T, n_envs), dtype=torch.int16), "shaped": torch.empty((T, n_envs, 2), dtype=torch.int8),
                     "done": torch.empty((T, n_envs), dtype=torch.uint8)}
            for d in dense.values():
                d.zero_()  # first touch on this rank's NUMA node, outside the timed region
        else:
            h_actions = torch.empty((T, n_envs, 2), dtype=pipe.act_dtype, pin_memory=True)
            h_actions.copy_(actions)
        env.reset()
        n_thr = max(1, host["bound_cpus"])
        overflow = [0]

        def finish(p_):
            """Pass p_ = (host tensors, ticket, dense-backup set) has been submitted: wait for it, expand it."""
            p_[1].synchronize()
            if expand:
                if stream:
                    pipe.expand(p_[0], codes_set=p_[2], out=dense, n_threads=n_thr)
                    overflow[0] += pipe.last_overflow
                else:
                    env.expand_codes(p_[0][3], out=dense, n_threads=n_thr)

        def passes_e2e(k):
            """k passes back to back, as a collection loop runs them: pass i+1 is submitted before pass i has
            drained (two pinned output sets), and with `expand` the host rebuilds pass i's arrays meanwhile."""
            prev = None
            for _ in range(k):
                h_, tk_ = pipe.run(h_actions, wait=False)
                cur_ = (h_, tk_, getattr(pipe, "_last_set", 0))
                if prev is not None:
                    finish(prev)
                prev = cur_
            finish(prev)
            pipe.join()
            return prev[0]

        passes_e2e(2)
        torch.cuda.synchronize(dev)
        D.barrier()
        k_e2e = max(3, min(args.steps, 8))
        overflow[0] = 0
        t0 = time.perf_counter()
        h_out = passes_e2e(k_e2e)
        torch.cuda.synchronize(dev)
        e2e_ms = (time.perf_counter() - t0) * 1e3
        D.barrier()
        _, e2e_max_ms, _ = D.reduce_counters(0, e2e_ms, 0, device=dev)
        if codes and expand:
            sparse_host = dense["sparse"]
        elif stream:
            sparse_host = pipe.expand(h_out, shaped=False, done=False)["sparse"]
        elif codes:
            sparse_host = env.expand_codes(h_out[3], shaped=False, done=False)["sparse"]
        else:
            sparse_host = h_out[0]
        exp_txt = ", expanded to dense int16 sparse / int8x2 shaped / uint8 done arrays by %d host threads inside the timed region" % n_thr if expand else ""
        what = {"stream": "a sparse event stream: per transition one warp-vote lane mask per 32 environments + the non-zero code words, %d value "
                          "slots per group and chunk (lossless; an overflowing group falls back to the dense words kept on the device)%s" % (pipe.stream_cap, exp_txt),
                "codes": "both agents' event codes + done + reward-grant bits in ONE int16 per env-step (lossless: rewards are table lookups of "
                         "the codes)%s" % exp_txt,
                "packed": "sparse int16 + shaped int8x2 + both agents' event codes and done in one int16 (lossless, wire.decode_event_codes)",
                "narrow": "sparse int16 / shaped int8 / done uint8 / events int32", "int32": "sparse/shaped/done/events int32"}[fmt]
        pipe.close()
        r = {"value": float(n_envs) * T * k_e2e * world / (e2e_max_ms * 1e-3), "unit": "env-steps/s",
             "h2d_bytes_per_step": pipe.h2d_bytes_per_step * T, "d2h_bytes_per_step": pipe.d2h_bytes_per_step * T,
             "steps": k_e2e, "ms_per_step": e2e_max_ms / k_e2e,
             "api": "overcooked_ai_b200.batched.HostRolloutPipeline(%s).run: pinned host actions (%s) in, %s out, "
                    "%d-transition chunks, H2D / fused rollout kernel / D2H on three streams, successive passes submitted back to back "
                    "(two pinned output sets; every pass's copies, its expansion and its completion are inside the timed region)"
                    % (fmt, "one uint8 per joint action" if codes else "uint8" if narrow else "int32", what, chunk),
             "host_threads": n_thr if expand else 0, "checksum_sparse": int(sparse_host.sum(dtype=torch.int64).item())}
        if stream:
            r["stream_overflows"] = overflow[0]
        return r

    def guarded(fn, *a_, **k_):
        """An optional leg must not cost the run its JSON line: a failure (the same on every rank: same code, same
        shapes) is reported in place of the leg's numbers."""
        try:
            return fn(*a_, **k_)
        except Exception as e:  # noqa: BLE001
            import traceback
            traceback.print_exc()
            return {"error": repr(e)[:300]}

    e2e = None
    if not args.no_e2e:
        if env.narrow_ok():
            e2e = run_e2e("stream", expand=True)             # headline: dense reward / done arrays in host memory
            e2e["event_stream_only"] = guarded(run_e2e, "stream")     # what crosses PCIe, left as the sparse stream
            e2e["code_words_expanded"] = guarded(run_e2e, "codes", expand=True)  # round 1's format: one dense int16 word per env-step
            e2e["int32_formats"] = guarded(run_e2e, "int32")          # the reference arm's own 32-bit formats (8 B in, 24 B out)
        else:
            e2e = run_e2e("int32")
        e2e["host_placement"] = host

    # ---- short legs of the other BASELINE configs (each: K5 value, roofline, sampled CPU replay) ----
    configs = {}
    if not args.no_configs and args.workload == "config2" and not args.envs:
        del out_t, out, actions, env
        torch.cuda.empty_cache()
        for name in ("config3", "config4", "target2e20"):
            configs[name] = guarded(lambda: engine_leg(name, dev, rank, world, seed, 3, 3, peak, peak_src, clocks=clocks)[0])
            torch.cuda.empty_cache()
        configs["config5"] = guarded(policy_leg, dev, rank, world, seed, 2, 1)

    if rank != 0:
        return

    k1_launch_s = k1_ms * 1e-3 / (k1_steps * T)
    k1_bytes = 2 * 4 * S + 32
    roofline_k1 = {
        "bound": "hbm", "kernel": "ovc::step_kernel<S=%d> K1: one transition per launch (ovc_step), 400 launches per CUDA graph" % S,
        "achieved": n_envs * k1_bytes / k1_launch_s / 1e9, "peak": peak, "unit": "GB/s", "frac": n_envs * k1_bytes / k1_launch_s / 1e9 / peak,
        "peak_source": peak_src, "algorithmic_bytes_per_env_step": k1_bytes, "env_steps_per_launch": n_envs, "avg_launch_us": k1_launch_s * 1e6,
        "env_steps_per_s_per_gpu": n_envs / k1_launch_s,
        "note": "SURVEY 8(d): record read + written, 8 B actions, 24 B outputs per env-step; at this batch size the state (%.1f MB) and the "
                "outputs are L2 resident, so DRAM traffic is below the algorithmic bytes" % (n_envs * S * 4 / 1e6),
    }
    line = {
        "metric": METRIC, "value": head["value"], "unit": "env-steps/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": head["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "int32", "data": "synthetic",
        "config": {
            "workload": head["workload"], "state_words": S, "mode": "rollout", "io": args.io,
            "parallelism": "env-index sharding x%d, no data-path collective" % world,
            "l2": "per bench step the action trace + outputs (%.0f MB) stream through HBM and exceed the %.0f MB L2; the %.1f MB state tensor "
                  "is the carried value (on chip for the whole launch)" % (n_envs * T * 32 / 1e6, torch.cuda.get_device_properties(dev).L2_cache_size / 1e6,
                                                                          n_envs * S * 4 / 1e6),
        },
        "clocks": clocks, "e2e": e2e, "gpu_launches": head["gpu_launches"], "roofline": head["roofline"], "roofline_k1": roofline_k1,
        "spot_check": head["spot_check"], "episode_sparse_reward_sum": head["sparse_reward_sum"],
    }
    if configs:
        line["configs"] = configs
    if not args.no_cpu:
        os.sched_setaffinity(0, set(host_affinity))  # the CPU arm gets every CPU the process may use, like --impl reference
        line["cpu_baseline"] = cpu_baseline(layouts, horizon)
    emit(line)


if __name__ == "__main__":
    try:
        main()
    finally:
        try:
            import torch.distributed as _d

            if _d.is_available() and _d.is_initialized():
                _d.destroy_process_group()
        except Exception:
            pass
