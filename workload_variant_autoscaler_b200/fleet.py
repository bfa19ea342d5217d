"""Flat SoA image of ``config.SystemSpec`` — the data layout that crosses the C ABI.

``Fleet.from_spec`` performs the joins that ``System.SetFromSpec``
(pkg/core/system.go:82-194) performs with Go maps: accelerator / model / service-class
names become dense ids, ``(model, accelerator)`` perf rows become an ``[M, A]`` table,
every server is joined with its service-class target.  The dict layout it accepts is
the JSON form of ``config.SystemSpec`` (pkg/config/types.go:11-155, same keys).
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from . import _abi
from ._abi import ACC_NONE, ACC_UNKNOWN

DEFAULT_SERVICE_CLASS = "Free"       # pkg/config/defaults.go:24
DEFAULT_LOW_PRIORITY = 100           # defaults.go:27
DEFAULT_HIGH_PRIORITY = 1            # defaults.go:30


def _i32(x):
    return np.ascontiguousarray(x, dtype=np.int32)


@dataclass
class Fleet:
    # accelerators [A]
    acc_cost: np.ndarray
    acc_multiplicity: np.ndarray
    acc_type: np.ndarray
    # accelerator types [T]
    type_capacity: np.ndarray
    # perf [M, A]
    perf_present: np.ndarray
    perf_alpha: np.ndarray
    perf_beta: np.ndarray
    perf_gamma: np.ndarray
    perf_delta: np.ndarray
    perf_acc_count: np.ndarray
    perf_max_batch: np.ndarray
    perf_at_tokens: np.ndarray
    # servers [S]
    srv_model: np.ndarray
    srv_priority: np.ndarray
    srv_has_target: np.ndarray
    srv_slo_itl: np.ndarray
    srv_slo_ttft: np.ndarray
    srv_slo_tps: np.ndarray
    srv_keep_acc: np.ndarray
    srv_min_replicas: np.ndarray
    srv_max_batch: np.ndarray
    srv_arrival_rpm: np.ndarray
    srv_in_tokens: np.ndarray
    srv_out_tokens: np.ndarray
    srv_cur_acc: np.ndarray
    srv_cur_replicas: np.ndarray
    srv_cur_cost: np.ndarray
    # optimizer spec
    unlimited: bool = True
    delayed_best_effort: bool = False
    saturation_policy: int = _abi.SAT_NONE
    max_queue_to_batch_ratio: int = 10     # config.MaxQueueToBatchRatio
    accel_penalty_factor: float = 0.1      # config.AccelPenaltyFactor
    # names (not part of the ABI; for reading results back)
    acc_names: list = field(default_factory=list)
    model_names: list = field(default_factory=list)
    server_names: list = field(default_factory=list)
    type_names: list = field(default_factory=list)

    # the array columns by element type (bench.py counts the fleet's bytes over these)
    _F32, _I32, _U8 = (tuple(n for n, dt, _ in _abi.FLEET_COLUMNS if dt is t) for t in (np.float32, np.int32, np.uint8))

    def __post_init__(self):
        for n, dt, _ in _abi.FLEET_COLUMNS:
            setattr(self, n, np.ascontiguousarray(getattr(self, n), dtype=dt))
        A = self.n_acc
        for n, _, length in _abi.FLEET_COLUMNS:
            if length == "MA":
                a = getattr(self, n)
                assert a.size % max(A, 1) == 0, n
                setattr(self, n, a.reshape(-1, A) if A else a.reshape(0, 0))

    @property
    def n_acc(self) -> int:
        return int(self.acc_cost.shape[0])

    @property
    def n_types(self) -> int:
        return int(self.type_capacity.shape[0])

    @property
    def n_models(self) -> int:
        return int(self.perf_present.shape[0])

    @property
    def n_servers(self) -> int:
        return int(self.srv_model.shape[0])

    def as_c(self) -> _abi.FleetC:
        """ctypes ``wva_fleet`` viewing this object's arrays (keep ``self`` alive)."""
        # building ~45 ctypes pointers costs more than the rest of a small solve's host path: the struct is
        # cached and reused while the very same array objects are still attached (in-place edits keep it valid)
        names = [n for n, _, _ in _abi.FLEET_COLUMNS]
        arrs = [getattr(self, n) for n in names]
        cache = self.__dict__.get("_c_cache")
        if cache is not None and all(a is b for a, b in zip(cache[0], arrs)):
            c = cache[1]
        else:
            p = _abi.ptr
            c = _abi.FleetC()
            for n, a in zip(names, arrs):
                setattr(c, n, p(a))
            self.__dict__["_c_cache"] = (arrs, c)
        c = _abi.FleetC.from_buffer_copy(c)  # callers may edit their struct; the cached one stays pristine
        c.n_acc, c.n_types, c.n_models, c.n_servers = self.n_acc, self.n_types, self.n_models, self.n_servers
        c.unlimited = 1 if self.unlimited else 0
        c.delayed_best_effort = 1 if self.delayed_best_effort else 0
        c.saturation_policy = int(self.saturation_policy)
        c.tun.max_queue_to_batch_ratio = int(self.max_queue_to_batch_ratio)
        c.tun.accel_penalty_factor = float(np.float32(self.accel_penalty_factor))
        return c

    def shard(self, rank: int, world: int) -> "Fleet":
        """Servers ``rank::world`` with the (small) accelerator / model tables replicated.

        Unlimited mode is separable per server (pkg/solver/solver.go:63-79), so shards
        need no data-path exchange; winners are all-gathered afterwards.
        """
        idx = np.arange(self.n_servers)[rank::world]
        return self.take_servers(idx)

    def take_servers(self, idx) -> "Fleet":
        kw = {}
        for n in self.__dataclass_fields__:
            v = getattr(self, n)
            if n.startswith("srv_"):
                kw[n] = v[idx].copy()
            elif n == "server_names":
                kw[n] = [v[i] for i in idx] if v else []
            else:
                kw[n] = v.copy() if isinstance(v, np.ndarray) else v
        return Fleet(**kw)

    def apply_winners(self, winners) -> "Fleet":
        """A copy of the fleet whose current allocation is advanced by one reconcile (``Server.ApplyDesiredAlloc``,
        pkg/core/server.go:157-161): a feasible winner's (accelerator, replicas, cost) becomes ``srv_cur_*``, and a
        server without one keeps its current allocation.  ``winners``: S records, an ``Allocs`` or a structured
        array with ``feasible`` / ``acc`` / ``replicas`` / ``cost`` fields (e.g. one tick of ``workload_trace``)."""
        def col(k):
            c = winners[k] if isinstance(winners, np.ndarray) else getattr(winners, k)
            if len(c) != self.n_servers:
                raise ValueError(f"winners must hold {self.n_servers} records, got {len(c)}")
            return np.asarray(c)
        f = self.take_servers(np.arange(self.n_servers))
        won = col("feasible") != 0
        f.srv_cur_acc[won] = col("acc")[won]
        f.srv_cur_replicas[won] = col("replicas")[won]
        f.srv_cur_cost[won] = col("cost")[won]
        return f

    # ------------------------------------------------------------------
    @staticmethod
    def from_spec(spec: dict, *, max_queue_to_batch_ratio: int = 10, accel_penalty_factor: float = 0.1) -> "Fleet":
        """Pack the JSON form of ``config.SystemSpec`` (a dict) into a Fleet."""
        accs = spec.get("acceleratorData", {}).get("accelerators", []) or []
        acc_names, acc_idx = [], {}
        for a in accs:  # AddAcceleratorFromSpec replaces on duplicate name (system.go:99-101)
            if a["name"] in acc_idx:
                continue
            acc_idx[a["name"]] = len(acc_names)
            acc_names.append(a["name"])
        last = {a["name"]: a for a in accs}
        A = len(acc_names)
        type_names, type_idx = [], {}
        for n in acc_names:
            t = last[n].get("type", "")
            if t not in type_idx:
                type_idx[t] = len(type_names)
                type_names.append(t)
        caps = {c["type"]: int(c["count"]) for c in (spec.get("capacityData", {}).get("count", []) or [])}
        for t in caps:
            if t not in type_idx:
                type_idx[t] = len(type_names)
                type_names.append(t)
        type_capacity = [caps.get(t, 0) for t in type_names]

        perf = spec.get("modelData", {}).get("models", []) or []
        model_names, model_idx = [], {}
        for pd in perf:
            if pd["name"] not in model_idx:
                model_idx[pd["name"]] = len(model_names)
                model_names.append(pd["name"])
        M = len(model_names)
        present = np.zeros((M, A), np.uint8)
        alpha = np.zeros((M, A), np.float32)
        beta = np.zeros((M, A), np.float32)
        gamma = np.zeros((M, A), np.float32)
        delta = np.zeros((M, A), np.float32)
        acc_count = np.ones((M, A), np.int32)
        max_batch = np.zeros((M, A), np.int32)
        at_tokens = np.zeros((M, A), np.int32)
        for pd in perf:  # AddPerfDataFromSpec (model.go:46-57); perf for unknown accs is unreachable
            m = model_idx[pd["name"]]
            if pd["acc"] not in acc_idx:
                continue
            a = acc_idx[pd["acc"]]
            present[m, a] = 1
            alpha[m, a] = pd.get("decodeParms", {}).get("alpha", 0.0)
            beta[m, a] = pd.get("decodeParms", {}).get("beta", 0.0)
            gamma[m, a] = pd.get("prefillParms", {}).get("gamma", 0.0)
            delta[m, a] = pd.get("prefillParms", {}).get("delta", 0.0)
            acc_count[m, a] = pd.get("accCount", 0)
            max_batch[m, a] = pd.get("maxBatchSize", 0)
            at_tokens[m, a] = pd.get("atTokens", 0)

        classes = {}
        for sc in spec.get("serviceClassData", {}).get("serviceClasses", []) or []:
            prio = int(sc.get("priority", 0))
            if prio < DEFAULT_HIGH_PRIORITY or prio > DEFAULT_LOW_PRIORITY:  # serviceclass.go:28-31
                prio = DEFAULT_LOW_PRIORITY
            targets = {}
            for mt in sc.get("modelTargets", []) or []:
                targets[mt["model"]] = (mt.get("slo-itl", 0.0), mt.get("slo-ttft", 0.0), mt.get("slo-tps", 0.0))
            classes[sc["name"]] = (prio, targets)

        servers = {}
        order = []
        for sv in spec.get("serverData", {}).get("servers", []) or []:
            if sv["name"] not in servers:
                order.append(sv["name"])
            servers[sv["name"]] = sv
        S = len(order)
        cols = {k: [] for k in ("model", "priority", "has_target", "itl", "ttft", "tps", "keep", "minrep", "maxb",
                                "rate", "intok", "outtok", "cacc", "crep", "ccost")}
        for name in order:
            sv = servers[name]
            cls = sv.get("class", "") or DEFAULT_SERVICE_CLASS  # server.go:35-38
            cur = sv.get("currentAlloc", {}) or {}
            load = cur.get("load", {}) or {}
            cols["model"].append(model_idx.get(sv.get("model", ""), -1))
            if cls in classes:
                prio, targets = classes[cls]
                t = targets.get(sv.get("model", ""))
            else:
                prio, t = DEFAULT_LOW_PRIORITY, None
            cols["priority"].append(prio)
            cols["has_target"].append(1 if t is not None else 0)
            cols["itl"].append(t[0] if t else 0.0)
            cols["ttft"].append(t[1] if t else 0.0)
            cols["tps"].append(t[2] if t else 0.0)
            cols["keep"].append(1 if sv.get("keepAccelerator", False) else 0)
            cols["minrep"].append(int(sv.get("minNumReplicas", 0)))
            cols["maxb"].append(int(sv.get("maxBatchSize", 0)))
            cols["rate"].append(load.get("arrivalRate", 0.0))
            cols["intok"].append(int(load.get("avgInTokens", 0)))
            cols["outtok"].append(int(load.get("avgOutTokens", 0)))
            cname = cur.get("accelerator", "") or ""
            cols["cacc"].append(ACC_NONE if cname == "" else acc_idx.get(cname, ACC_UNKNOWN))
            cols["crep"].append(int(cur.get("numReplicas", 0)))
            cols["ccost"].append(cur.get("cost", 0.0))

        opt = spec.get("optimizerData", {}).get("optimizer", {}) or {}
        return Fleet(
            acc_cost=[last[n].get("cost", 0.0) for n in acc_names],
            acc_multiplicity=[int(last[n].get("multiplicity", 0)) for n in acc_names],
            acc_type=[type_idx[last[n].get("type", "")] for n in acc_names],
            type_capacity=type_capacity,
            perf_present=present, perf_alpha=alpha, perf_beta=beta, perf_gamma=gamma, perf_delta=delta,
            perf_acc_count=acc_count, perf_max_batch=max_batch, perf_at_tokens=at_tokens,
            srv_model=cols["model"], srv_priority=cols["priority"], srv_has_target=cols["has_target"],
            srv_slo_itl=cols["itl"], srv_slo_ttft=cols["ttft"], srv_slo_tps=cols["tps"],
            srv_keep_acc=cols["keep"], srv_min_replicas=cols["minrep"], srv_max_batch=cols["maxb"],
            srv_arrival_rpm=cols["rate"], srv_in_tokens=cols["intok"], srv_out_tokens=cols["outtok"],
            srv_cur_acc=cols["cacc"], srv_cur_replicas=cols["crep"], srv_cur_cost=cols["ccost"],
            unlimited=bool(opt.get("unlimited", False)),
            delayed_best_effort=bool(opt.get("delayedBestEffort", False)),
            saturation_policy=_abi.SAT_BY_NAME.get(opt.get("saturationPolicy", ""), _abi.SAT_NONE),
            max_queue_to_batch_ratio=max_queue_to_batch_ratio, accel_penalty_factor=accel_penalty_factor,
            acc_names=acc_names, model_names=model_names, server_names=order, type_names=type_names,
        )


@dataclass
class Grid:
    batch: np.ndarray
    replicas: np.ndarray

    def __post_init__(self):
        self.batch = _i32(self.batch)
        self.replicas = _i32(self.replicas)

    def as_c(self) -> _abi.GridC:
        cache = self.__dict__.get("_c_cache")
        if cache is not None and cache[0] is self.batch and cache[1] is self.replicas:
            return cache[2]
        c = _abi.GridC(int(self.batch.size), _abi.ptr(self.batch), int(self.replicas.size), _abi.ptr(self.replicas))
        self.__dict__["_c_cache"] = (self.batch, self.replicas, c)
        return c


# ----------------------------------------------------------------------------
# Synthetic fleets (SURVEY.md §8d). Seeded PCG64; all values float32-rounded.
# ----------------------------------------------------------------------------

SLO_CLASSES = ((24.0, 500.0), (80.0, 500.0), (150.0, 1500.0), (200.0, 2000.0))
ACC_COSTS = (23.0, 40.0, 65.0, 80.0, 30.0, 55.0, 95.0, 120.0)


def synth_fleet(n_servers: int, n_acc: int, *, seed: int = 42, n_models: int | None = None,
                keep_accelerator: bool = False, max_batch_choices=(4, 8, 16, 32, 64, 128, 256, 512),
                zero_load_frac: float = 0.05, tps_frac: float = 0.10, server_batch: bool = True) -> Fleet:
    """Seeded N-model x M-accelerator fleet with the distributions of SURVEY.md §8d config 2."""
    rng = np.random.Generator(np.random.PCG64(seed))
    S, A = n_servers, n_acc
    M = n_models or n_servers
    h100_like = rng.random((M, A)) < 0.5
    alpha = rng.uniform(5.0, 25.0, (M, A))
    beta = np.where(h100_like, rng.uniform(0.03, 0.05, (M, A)), rng.uniform(0.02, 0.8, (M, A)))
    gamma = rng.uniform(0.0, 250.0, (M, A))
    delta = np.exp(rng.uniform(np.log(1e-4), np.log(0.1), (M, A)))
    acc_count = rng.choice([1, 2, 4, 8], (M, A))
    max_batch = rng.choice(list(max_batch_choices), (M, A))
    cost = np.array([ACC_COSTS[i % len(ACC_COSTS)] for i in range(A)], np.float32)

    arrival = np.exp(rng.uniform(np.log(1.0), np.log(5000.0), S))
    arrival[rng.random(S) < zero_load_frac] = 0.0
    in_tok = rng.integers(16, 2049, S)
    out_tok = rng.integers(16, 1025, S)
    slo = rng.integers(0, len(SLO_CLASSES), S)
    tps = np.where(rng.random(S) < tps_frac, rng.choice([500.0, 2000.0], S), 0.0)
    cur_acc = rng.integers(-1, A, S)  # -1 = "" (no current accelerator)
    cur_rep = np.where(cur_acc >= 0, rng.integers(1, 9, S), 0)
    srv_model = np.arange(S) % M
    # Production sets the batch size per server from the VA profile
    # (internal/utils/utils.go:296-307); AtTokens is never set there (SURVEY.md hard part f).
    srv_max_batch = rng.choice(list(max_batch_choices), S) if server_batch else np.zeros(S)
    cur_cost = np.where(cur_acc >= 0,
                        cost[np.maximum(cur_acc, 0)] * acc_count[srv_model, np.maximum(cur_acc, 0)] * cur_rep, 0.0)
    return Fleet(
        acc_cost=cost, acc_multiplicity=np.ones(A), acc_type=np.arange(A), type_capacity=np.full(A, 1 << 20),
        perf_present=np.ones((M, A)), perf_alpha=alpha, perf_beta=beta, perf_gamma=gamma, perf_delta=delta,
        perf_acc_count=acc_count, perf_max_batch=max_batch, perf_at_tokens=np.full((M, A), 512),
        srv_model=srv_model, srv_priority=np.where(slo < 2, 1, 10), srv_has_target=np.ones(S),
        srv_slo_itl=[SLO_CLASSES[i][0] for i in slo], srv_slo_ttft=[SLO_CLASSES[i][1] for i in slo],
        srv_slo_tps=tps, srv_keep_acc=np.full(S, 1 if keep_accelerator else 0), srv_min_replicas=np.ones(S),
        srv_max_batch=srv_max_batch, srv_arrival_rpm=arrival, srv_in_tokens=in_tok, srv_out_tokens=out_tok,
        srv_cur_acc=cur_acc, srv_cur_replicas=cur_rep, srv_cur_cost=cur_cost, unlimited=True,
        acc_names=[f"acc{i}" for i in range(A)], model_names=[f"model{i}" for i in range(M)],
        server_names=[f"srv{i}:ns" for i in range(S)], type_names=[f"type{i}" for i in range(A)],
    )


def config1_fleet(arrival_rpm: float, in_tok: int, out_tok: int) -> Fleet:
    """BASELINE configs[0]: the single VariantAutoscaling of deploy/examples/vllm-emulator
    (vllme-variantautoscaling.yaml:26-37: A100 alpha 20.58 beta 0.41 gamma 5.2 delta 0.1, maxBatch 4;
    deploy/configmap-*.yaml: A100 cost 40.00, Premium slo-tpot 24 / slo-ttft 500), production flags
    (unlimited, keepAccelerator, minReplicas 1: internal/utils/utils.go:170-173,290)."""
    spec = {
        "acceleratorData": {"accelerators": [{"name": "A100", "type": "NVIDIA-A100-PCIE-80GB", "multiplicity": 1,
                                              "cost": 40.0}]},
        "modelData": {"models": [{"name": "default/default", "acc": "A100", "accCount": 1, "maxBatchSize": 4,
                                  "decodeParms": {"alpha": 20.58, "beta": 0.41},
                                  "prefillParms": {"gamma": 5.2, "delta": 0.1}}]},
        "serviceClassData": {"serviceClasses": [{"name": "Premium", "priority": 1, "modelTargets": [
            {"model": "default/default", "slo-itl": 24.0, "slo-ttft": 500.0}]}]},
        "serverData": {"servers": [{"name": "vllme-deployment:llm-d-sim", "model": "default/default",
                                    "class": "Premium", "keepAccelerator": True, "minNumReplicas": 1,
                                    "maxBatchSize": 4,
                                    "currentAlloc": {"accelerator": "A100", "numReplicas": 1, "cost": 40.0,
                                                     "load": {"arrivalRate": arrival_rpm, "avgInTokens": in_tok,
                                                              "avgOutTokens": out_tok}}}]},
        "optimizerData": {"optimizer": {"unlimited": True}},
    }
    return Fleet.from_spec(spec)


CONFIG1_LOADS = (0.0, 60.0, 480.0, 960.0, 1440.0)
CONFIG1_TOKENS = ((0, 278), (128, 128))  # emulator through the collector; and the 128/128 variant


def config2_grid(n_batch: int = 256, n_replicas: int = 64) -> Grid:
    """BASELINE config 2: batch sizes 1..B, replica levels 1..R."""
    return Grid(np.arange(1, n_batch + 1), np.arange(1, n_replicas + 1))
