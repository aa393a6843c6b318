"""CPU: the decisions of the three in-flight schedule oracles (tests/inflight_oracle.py, kv_pool_oracle.py, prefix_cache_oracle.py) on the
seeded scripts the oracle and GPU tests drive, against a recorded trace (tests/golden/inflight_schedule_trace.npz, written by
tests/golden/make_golden_inflight_schedule.py).  The GPU tests compare the kernel with the oracles, so a change made to both alike passes
them; this trace pins the decisions themselves: plans, row states, outputs, victims, blocked starts, evictions, duplicates and LRU order.

After every schedule call each component of the state is digested separately, so that a mismatch names its script, step and component.
The trace is never regenerated to make this test pass: a mismatch means a rule changed."""
import hashlib
import os

import numpy as np
import pytest

from tests.inflight_oracle import InflightOracle
from tests.kv_pool_oracle import KvPoolOracle, min_pages
from tests.prefix_cache_oracle import PrefixCacheOracle
from tests import test_oracle_inflight, test_oracle_kv_pool, test_oracle_prefix_cache

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inflight_schedule_trace.npz")


def _digest(x) -> int:
    return int.from_bytes(hashlib.blake2b(repr(x).encode(), digest_size=4).digest(), "little")


def _components(o: InflightOracle, plan) -> dict:
    c = dict(plan=plan,
             rows=(o.phase, o.row_req, o.done, o.adm, o.finished, o.prompt_lens, o.seq_lens, o.start_pos),
             outputs=(sorted(o.outputs.items()), o.ring, o.head, o.retired, o.admitted))
    if isinstance(o, KvPoolOracle):
        c.update(pool=(o.free, o.row_pages, o.target, o.counters(), sorted(o.tables.items())), events=sorted(o.events.items()))
    if isinstance(o, PrefixCacheOracle):
        c.update(cache=(o.ref, o.state, o.epoch, o.key, o.reg, o.halted, o.lru, sorted(o.index.items()), o.cache_counters()))
    return c


def _inflight(seed):
    def run(rec):
        test_oracle_inflight._run_script(seed, *test_oracle_inflight._config(seed), check=rec)
    return run


def _pool(seed, B, Q, C, ctx, T, n, P, blocks, layers, vocab=50):
    def run(rec):
        o = KvPoolOracle(B, Q, C, T, ctx, P, blocks, layers=layers)
        test_oracle_kv_pool._drive([o], seed, B, Q, C, ctx, T, n, vocab=vocab, check=lambda step, plans: rec(o, plans[0]))
    return run


def _cache(seed, B, Q, C, ctx, T, n, P, blocks, layers, vocab=50):
    def run(rec):
        o = PrefixCacheOracle(B, Q, C, T, ctx, P, blocks, layers=layers)
        test_oracle_prefix_cache.drive_shared([o], seed, B, Q, C, ctx, T, n, vocab=vocab, check=lambda step, plans: rec(o, plans[0]))
    return run


def scripts() -> dict:
    """name -> run(record): every script drives one oracle and calls record(oracle, plan) after each schedule call."""
    out = {f"inflight_random_{s}": _inflight(s) for s in range(12)}
    for s in range(16):  # test_smallest_pool_finishes_and_conserves_pages
        B, Q, C, ctx, T, n = test_oracle_kv_pool._config(s)
        P = min_pages(ctx, T)
        out[f"pool_smallest_{s}"] = _pool(s, B, Q, C, ctx, T, n, P, P, 2)
    out["pool_every_event"] = _pool(31, 6, 7, 40, 150, 60, 40, 7, min_pages(150, 60), 1, vocab=400)
    out["pool_gpu"] = _pool(31, 6, 7, 40, 150, 60, 40, 7, min_pages(150, 60) + 1, 3, vocab=400)  # test_gpu_kv_pool's configuration
    for s in range(16):  # test_shared_scripts_keep_the_invariants (2 layers) and test_shared_scripts_hit_evict_and_preempt (1 layer)
        B, Q, C, ctx, T, n, scale = test_oracle_prefix_cache._shared_config(s)
        P, blocks = min_pages(ctx, T) * scale, min_pages(ctx, T) + 1
        out[f"cache_shared_{s}"] = _cache(s, B, Q, C, ctx, T, n, P, blocks, 2)
        out[f"cache_hit_{s}"] = _cache(s, B, Q, C, ctx, T, n, P, blocks, 1)
    out["cache_gpu"] = _cache(11, 5, 7, 64, 200, 40, 30, min_pages(200, 40) * 2, min_pages(200, 40) + 1, 2)  # test_gpu_prefix_cache's
    return out


def trace(run) -> dict:
    """component -> 32-bit digests, one per schedule call."""
    rec: dict = {}

    def record(o, plan):
        for k, v in _components(o, plan).items():
            rec.setdefault(k, []).append(_digest(v))

    run(record)
    return {k: np.array(v, dtype=np.uint32) for k, v in rec.items()}


SCRIPTS = scripts()


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", list(SCRIPTS))
def test_schedule_decisions_match_the_trace(golden, name):
    got = trace(SCRIPTS[name])
    want = {k.split(":", 1)[1]: v for k, v in golden.items() if k.split(":", 1)[0] == name}
    assert sorted(got) == sorted(want), (name, sorted(got), sorted(want))
    steps = len(want["plan"])
    for k in want:
        assert len(got[k]) == steps, f"{name}: {len(got[k])} schedule calls, the trace has {steps}"
    for step in range(steps):
        bad = [k for k in sorted(want) if got[k][step] != want[k][step]]
        assert not bad, f"{name}: step {step} differs in {bad}"
