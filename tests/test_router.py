"""Router parity: the reference's own tables (internal/loadbalancer/load_balancer_test.go) replayed
against (a) the Python oracle and (b) the C++ router behind the C ABI.  CPU only."""
import random
import threading

import pytest

from kubeai_b200 import lib
from kubeai_b200.router import LEAST_LOAD, PREFIX_HASH, DeadlineExceeded, Router
from oracle.router_oracle import Group
from oracle.weights import xxh64

A1, A2, B1, B2 = "10.0.0.1:8000", "10.0.0.2:8000", "10.0.0.3:8000", "10.0.0.4:8000"


def test_xxh64_known_answers():
    # SURVEY.md §7 step 1a (python-xxhash == cespare/xxhash Sum64) + XXH64 spec test vector for ""
    kat = {b"": 0xEF46DB3751D8E999, b"pod-a-10": 689047897566398072, b"pod-a-20": 8996271527020827053}
    l = lib()
    for s, h in kat.items():
        assert xxh64(s) == h
        assert l.b200_xxh64(s, len(s)) == h
    xxhash = pytest.importorskip("xxhash")
    rng = random.Random(1)
    for n in list(range(0, 70)) + [100, 255, 256, 1000]:
        s = bytes(rng.randrange(256) for _ in range(n))
        want = xxhash.xxh64(s).intdigest()
        assert xxh64(s) == want and l.b200_xxh64(s, n) == want, n


class OracleLB:
    """model -> Group, with the Go test's AwaitBestAddress / done-func shape."""

    def __init__(self, replication):
        self.rep, self.groups = replication, {}

    def reconcile(self, model, eps):
        self.groups.setdefault(model, Group(self.rep)).reconcile(eps)

    def add_in_flight(self, model, name, n):
        self.groups[model].add_in_flight(name, n)

    def pick(self, model, strategy, adapter, prefix, pct):
        g = self.groups.get(model)
        r = g.pick(strategy, adapter, prefix, pct) if g else None
        if r is None:
            raise DeadlineExceeded()
        addr, name = r
        return addr, (lambda: g.done(name))


class NativeLB:
    def __init__(self, replication):
        self.rep, self.groups = replication, {}

    def _g(self, model):
        if model not in self.groups:
            self.groups[model] = Router(self.rep)
        return self.groups[model]

    def reconcile(self, model, eps):
        self._g(model).reconcile_endpoints(eps)

    def add_in_flight(self, model, name, n):
        self._g(model).add_in_flight(name, n)

    def pick(self, model, strategy, adapter, prefix, pct):
        return self._g(model).await_best_address(strategy, adapter, prefix, pct, timeout_s=0.001)


IMPLS = [OracleLB, NativeLB]


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("strategy", [LEAST_LOAD, PREFIX_HASH])
def test_await_best_host_behavior(impl, strategy):
    """load_balancer_test.go:19-129"""
    cases = {
        "model only": ("my-model", "", {"pod1": dict(address=A1)}, A1),
        "model and adapter": ("my-model", "my-adapter",
                              {"pod1": dict(address=A1), "pod2": dict(address=A2, adapters={"my-adapter"})}, A2),
        "no matching model blocks until timeout": ("unknown-model", "", {"pod1": dict(address=A1)}, None),
        "no matching adapter blocks until timeout": ("my-model", "unknown-adapter", {"pod1": dict(address=A1)}, None),
    }
    for name, (model, adapter, eps, exp) in cases.items():
        lb = impl(1)
        lb.reconcile("my-model", eps)
        if exp is None:
            with pytest.raises(DeadlineExceeded):
                lb.pick(model, strategy, adapter, "", 125)
        else:
            addr, done = lb.pick(model, strategy, adapter, "", 125)
            done()
            assert addr == exp, name


def _run_steps(lb, strategy, pct, steps):
    done_funcs = {}
    for step in steps:
        counts = {}
        for _ in range(step.get("n", 0)):
            addr, done = lb.pick(step["model"], strategy, step.get("adapter", ""), step.get("prefix", ""), pct)
            done_funcs.setdefault(addr, []).append(done)
            counts[addr] = counts.get(addr, 0) + 1
        if "expect" in step:
            assert counts == step["expect"], step["name"]
        for addr, k in step.get("complete", {}).items():
            for _ in range(k):
                done_funcs[addr].pop(0)()
    for ds in done_funcs.values():
        for d in ds:
            d()


@pytest.mark.parametrize("impl", IMPLS)
def test_least_load_strategy_table(impl):
    """load_balancer_test.go:177-257 — exact per-step address counts"""
    lb = impl(1)
    lb.reconcile("model-a", {"pod-a-1": dict(address=A1, adapters={"adapter-a-1"}),
                             "pod-a-2": dict(address=A2, adapters={"adapter-a-2"})})
    lb.reconcile("model-b", {"pod-b-1": dict(address=B1), "pod-b-2": dict(address=B2)})
    steps = [
        dict(name="first 2", model="model-a", n=2, expect={A1: 1, A2: 1}),
        dict(name="a lot more", model="model-a", n=100, expect={A1: 50, A2: 50}),
        dict(name="adapter-a-1", model="model-a", adapter="adapter-a-1", n=50, expect={A1: 50}),
        dict(name="without adapter goes to the other pod", model="model-a", n=52, expect={A1: 1, A2: 51}),
        dict(name="back to even", model="model-a", n=2, expect={A1: 1, A2: 1}),
        dict(name="complete some for pod-a-2", complete={A2: 10}),
        dict(name="now distributed to the other pod", model="model-a", n=12, expect={A1: 1, A2: 11}),
        dict(name="first requests to model-b", model="model-b", n=2, expect={B1: 1, B2: 1}),
    ]
    _run_steps(lb, LEAST_LOAD, 125, steps)


@pytest.mark.parametrize("impl", IMPLS)
def test_prefix_hash_strategy_table(impl):
    """load_balancer_test.go:259-369 incl. the load-threshold table at :299-346"""
    lb = impl(1)
    lb.reconcile("model-a", {"pod-a-1": dict(address=A1), "pod-a-2": dict(address=A2)})
    lb.reconcile("model-b", {"pod-b-1": dict(address=B1)})
    lb.add_in_flight("model-a", "pod-a-1", 10)
    lb.add_in_flight("model-a", "pod-a-2", 10)
    h1, h2 = "pod-a-10", "pod-a-20"      # chwblEndpointReplicaHashInput(name, 0)
    steps = [
        dict(name="first, preferring pod-a-1", model="model-a", prefix=h1, n=1, expect={A1: 1}),
        dict(name="20 more preferring pod-a-1", model="model-a", prefix=h1, n=20, expect={A1: 20}),
        dict(name="4 more preferring pod-a-1", model="model-a", prefix=h1, n=4, expect={A1: 3, A2: 1}),
        dict(name="preferring pod-a-2", model="model-a", prefix=h2, n=20, expect={A2: 20}),
        dict(name="model-b ring is separate", model="model-b", prefix=h2,
             n=100_000 if impl is NativeLB else 5_000, expect={B1: 100_000 if impl is NativeLB else 5_000}),
    ]
    _run_steps(lb, PREFIX_HASH, 150, steps)


def test_native_matches_oracle_on_random_traffic():
    """Same request stream, same endpoint churn -> identical choices (ring order, thresholds, wrap)."""
    rng = random.Random(42)
    for rep in (1, 7, 256):
        o, n = Group(rep), Router(rep)
        names = [f"gpu-{i}" for i in range(8)]
        live = {}
        outstanding = []
        for step in range(3000):
            if step % 400 == 0:
                k = rng.randrange(1, 9)
                live = {nm: dict(address=f"10.1.0.{i}:8000", adapters={"lora"} if i % 3 == 0 else set())
                        for i, nm in enumerate(rng.sample(names, k))}
                o.reconcile(live)
                n.reconcile_endpoints(live)
            strat = PREFIX_HASH if rng.random() < 0.7 else LEAST_LOAD
            adapter = "lora" if rng.random() < 0.2 else ""
            prefix = "héllo wörld %d" % rng.randrange(200)
            pct = rng.choice([100, 125, 150, 100000])
            exp = o.pick(strat, adapter, prefix, pct)
            if exp is None:
                with pytest.raises(DeadlineExceeded):
                    n.await_best_address(strat, adapter, prefix, pct, timeout_s=0)
                continue
            addr, done = n.await_best_address(strat, adapter, prefix, pct, timeout_s=0)
            assert addr == exp[0], (rep, step)
            outstanding.append((exp[1], done))
            if len(outstanding) > 40 or rng.random() < 0.3:
                nm, d = outstanding.pop(rng.randrange(len(outstanding)))
                o.done(nm)
                d()
        assert n.in_flight()[1] == o.total_in_flight


def test_parallel_accounting():
    """load_balancer_test.go:431-515: many concurrent picks, <=4 % imbalance, counters return to 0."""
    for strategy in (LEAST_LOAD, PREFIX_HASH):
        r = Router(256)
        r.reconcile_endpoints({"pod0": dict(address=A1), "pod1": dict(address=A2)})
        N, TH = 40_000, 16
        dones = [[] for _ in range(TH)]

        def work(t):
            rng = random.Random(t)
            for _ in range(N // TH):
                _, d = r.await_best_address(strategy, "", str(rng.randrange(100_000_000)), 100000, timeout_s=0.001)
                dones[t].append(d)

        th = [threading.Thread(target=work, args=(t,)) for t in range(TH)]
        [t.start() for t in th]
        [t.join() for t in th]
        e0, tot = r.in_flight("pod0")
        e1, _ = r.in_flight("pod1")
        assert tot == N and e0 + e1 == N
        assert abs(e0 - e1) / ((e0 + e1) / 2) * 100 < 4.0
        for ds in dones:
            for d in ds:
                d()
        assert r.in_flight("pod0") == (0, 0) and r.in_flight("pod1")[0] == 0


def test_blocked_request_wakes_when_endpoint_appears():
    """group.go:56-64,139-145: waiters are released by reconcileEndpoints' broadcast."""
    r = Router(16)
    got = {}

    def waiter():
        got["addr"], got["done"] = r.await_best_address(LEAST_LOAD, timeout_s=5.0)

    t = threading.Thread(target=waiter)
    t.start()
    import time
    time.sleep(0.05)
    assert "addr" not in got
    r.reconcile_endpoints({"gpu-0": dict(address="10.9.9.9:1")})
    t.join(5)
    assert got["addr"] == "10.9.9.9:1"
    # removed endpoints drain: done() after removal must not underflow the group total
    r.reconcile_endpoints({"gpu-1": dict(address="10.9.9.8:1")})
    got["done"]()
    assert r.in_flight()[1] == 0


def test_hash_lookup_metrics_follow_the_reference_instruments():
    """internal/metrics/metrics.go:19-26,51-76 emitted at balance_chwbl.go:24-26,58-61,74-80."""
    r = Router(1)
    r.reconcile_endpoints({"pod-a-1": dict(address=A1), "pod-a-2": dict(address=A2)})
    r.add_in_flight("pod-a-1", 10)
    r.add_in_flight("pod-a-2", 10)
    dones = [r.await_best_address(PREFIX_HASH, "", "pod-a-10", 150, timeout_s=0)[1] for _ in range(25)]
    m = r.metrics()
    # 25 lookups start at pod-a-1; 24 stay there (threshold table load_balancer_test.go:299-346), one walks to pod-a-2
    assert 'kubeai_inference_requests_hash_lookup_initial{endpoint="pod-a-1"} 25' in m
    assert 'kubeai_inference_requests_hash_lookup_final{endpoint="pod-a-1"} 24' in m
    assert 'kubeai_inference_requests_hash_lookup_final{endpoint="pod-a-2"} 1' in m
    assert 'kubeai_inference_requests_hash_lookup_iterations_bucket{le="1"} 24' in m
    assert 'kubeai_inference_requests_hash_lookup_iterations_bucket{le="2"} 25' in m
    assert "kubeai_inference_requests_hash_lookup_iterations_sum 26" in m and "hash_lookup_default{" not in m
    [d() for d in dones]


def test_closed_loop_least_load_is_sticky_like_prefix_hash():
    """A side finding of the live routing experiment (DESIGN.md §6): in a closed-loop load generator a conversation's next
    turn is issued when its previous turn finishes, i.e. on the endpoint that just lost one in-flight request — so LeastLoad
    keeps most conversations where their KV prefix is, without looking at the prefix.  Event simulation on the native
    router: 8 endpoints, 64 conversations of 12 turns, service times with jitter."""
    import heapq
    import random
    from kubeai_b200.router import LEAST_LOAD, PREFIX_HASH, Router

    def run(strategy):
        rng = random.Random(5)
        r = Router(replication=256)
        r.reconcile_endpoints({f"pod-{i}": {"address": f"gpu:{i}"} for i in range(8)})
        events, last, same, total = [], {}, 0, 0
        for c in range(64):
            heapq.heappush(events, (rng.random() * 0.01, c, 0, None))       # (time, conversation, turn, done of the previous turn)
        while events:
            t, c, turn, done = heapq.heappop(events)
            if done is not None:
                done()                                                      # the previous turn's request ends ...
            if turn == 12:
                continue
            addr, d = r.await_best_address(strategy, prefix=f"conversation {c:04d} first user message", mean_load_pct=125)
            if turn > 0:
                total += 1
                same += addr == last[c]
            last[c] = addr
            heapq.heappush(events, (t + 0.25 + 0.1 * rng.random(), c, turn + 1, d))    # ... and the next one starts at once
        assert r.in_flight()[1] == 0
        r.close()
        return same / total

    sticky_ll, sticky_ph = run(LEAST_LOAD), run(PREFIX_HASH)
    assert sticky_ph >= 0.97, sticky_ph           # CHWBL moves a conversation only when its endpoint is over the load bound
    assert sticky_ll >= 0.5, sticky_ll            # far above the 1/8 of a prefix-blind uniform choice (measured here: 0.987)
