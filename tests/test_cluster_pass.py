"""Frontier clustering pass (tlag_engine.cu, cluster_slice): every newly discovered level of 8192 states or more is
reordered, stably, by the key w[W-1] << 32 | w[W-2], through a sort on the key's dense rank among the level's distinct
keys and one gather back into the store.  On the sliced native kernels, for a scalar-form and an array-form model:

- every clustered level reads back ordered by (w[W-1], w[W-2]), and holds exactly the oracle's states of that level;
- sampled parent links point into the previous level;
- counts, per-level sizes and digests match the oracle with the rank set at its default size, with a rank set of
  4 slots (TLAG_RSET_SLOTS: it fills up and grows on every clustered level), and with the pass switched off
  (TLAG_NO_SORT=1).  Both are read when the engine is created."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from tla_rust_b200.compiled import load_compiled

# MCPaxos3_b3 is scalar form (W = 8, 8.2 M states), MCraft_t4l3 array form (W = 62, 11.3 M states); the level-by-level
# comparison with the oracle's states runs on the first `levels` levels of each (7 and 5 clustered levels)
CASES = [("MCPaxos3_b3", 18), ("MCraft_t4l3", 11)]
NAMES = [n for n, _ in CASES]


def _run(name, max_levels=0):
    """the sliced engine on `name`, to the fixpoint or for `max_levels` levels: (engine, per-level sizes, result)"""
    from tla_rust_b200.engine import V_RUNNING, Engine
    cm, init, exp, info = load_compiled(os.path.join(GOLDEN, name + ".tlagz"))
    e = Engine(cm, deadlock=info["deadlock"], native="sliced")
    e.seed(init)
    levels = [int(len(np.unique(init, axis=0)))]
    while not max_levels or len(levels) < max_levels:
        ws = e.step()
        if ws["expanded"]:
            levels.append(int(ws["discovered"]))
        if ws["verdict"] != V_RUNNING:
            break
    return e, levels, e.result()


def _expect(name):
    """the fixture's oracle record of the whole search: per-level sizes, (generated, distinct, depth), digest"""
    _, _, exp, _ = load_compiled(os.path.join(GOLDEN, name + ".tlagz"))
    o2 = exp["o2"]
    return o2["levels"], (o2["generated"], o2["distinct"], o2["depth"]), (o2["fp_xor"], o2["fp_sum"])


@pytest.mark.gpu
@pytest.mark.parametrize("name,max_levels", CASES)
def test_clustered_levels_are_ordered_by_key_and_hold_the_oracles_states(monkeypatch, name, max_levels):
    from oracle import cpu_engine
    monkeypatch.delenv("TLAG_RSET_SLOTS", raising=False)
    cm, init, _, info = load_compiled(os.path.join(GOLDEN, name + ".tlagz"))
    e, levels, r = _run(name, max_levels)
    o2 = cpu_engine.run(cm, init, n_threads=4, deadlock=info["deadlock"], max_states=r["distinct"] + 1024,
                        want_states=True, max_levels=max_levels)
    x, sm, gen = o2["level_digests"][max_levels - 1]
    assert levels == o2["levels"][:max_levels]
    assert (r["generated"], r["distinct"], r["depth"]) == (gen, sum(levels), max_levels)
    assert e.digest() == (x, sm)
    W = cm.W
    got = e.read_states(0, r["distinct"]).reshape(-1, W)
    ref = o2["states"].reshape(-1, W)
    rng = np.random.default_rng(7)
    clustered = 0
    start = 0
    prev = (0, 0)
    for size in levels:
        lvl = got[start:start + size]
        if size >= 8192:
            clustered += 1
            key = (lvl[:, W - 1].astype(np.uint64) << np.uint64(32)) | (lvl[:, W - 2].astype(np.uint64) if W >= 2 else 0)
            assert np.all(key[1:] >= key[:-1]), f"level of {size} states not ordered by its key"
        a = lvl[np.lexsort(lvl.T[::-1])]
        b = ref[start:start + size][np.lexsort(ref[start:start + size].T[::-1])]
        assert np.array_equal(a, b), f"level starting at {start}: state set differs from the oracle's"
        if start > 0:      # sampled links: the parent lies in the previous level, the row read with its link is the row
            for i in rng.choice(size, size=min(size, 200), replace=False):
                row, parent, _, _ = e.read_link(start + int(i))
                assert np.array_equal(np.asarray(row, dtype=np.uint32), lvl[i])
                assert prev[0] <= parent < prev[1], (start + int(i), parent, prev)
        prev = (start, start + size)
        start += size
    assert clustered >= 3
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_a_tiny_rank_set_grows_and_changes_nothing(monkeypatch, name):
    monkeypatch.setenv("TLAG_RSET_SLOTS", "4")
    want_levels, want_counts, want_digest = _expect(name)
    e, levels, r = _run(name)
    assert levels == want_levels
    assert (r["generated"], r["distinct"], r["depth"]) == want_counts
    assert e.digest() == want_digest
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_without_clustering_the_counts_and_digests_are_the_same(monkeypatch, name):
    monkeypatch.setenv("TLAG_NO_SORT", "1")
    monkeypatch.delenv("TLAG_RSET_SLOTS", raising=False)
    want_levels, want_counts, want_digest = _expect(name)
    e, levels, r = _run(name)
    assert levels == want_levels
    assert (r["generated"], r["distinct"], r["depth"]) == want_counts
    assert e.digest() == want_digest
    e.close()
