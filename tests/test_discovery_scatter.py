"""Discovery buffer (tlag_engine.cu: open_level, cluster_slice, k_cluster_gather): a level's new rows are appended to a
buffer of records [W words, parent, meta] and moved into the store when the level ends, stably sorted by key, or in
discovery order when the level is not clustered.

- On a box model of test_shapes (interpreter kernel, and the sliced kernels' staged appends), every stored row is its
  parent's state moved by +D in exactly one coordinate, with the model's one action in its meta word: parent and meta
  travel with the row; every level the pass sorts reads back in ascending key order.
- A violation that ends the search (its last level is not clustered) and keep_going leave the oracle's counts and
  digest; the last level is read back from the store.
- tlag_read_states and tlag_digest between tlag_p2p_level and tlag_advance_level (world size 1) see every row of the
  level still in the buffer."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from test_shapes import BY_NAME, _compiled, _spec, shapes_dir  # noqa: F401  (shapes_dir: fixture)
from tla_rust_b200.checker import compile_model, encode_states
from tla_rust_b200.compiled import load_compiled
from tla_rust_b200.front.spec import Model


def _clear(monkeypatch):
    for k in ("TLAG_TIGHT_HEADROOM", "TLAG_RSET_SLOTS", "TLAG_NO_SORT", "TLAG_SL_STAGE", "TLAG_SL_SKIPSELF"):
        monkeypatch.delenv(k, raising=False)


def _sorted_levels(rows, sizes, W):
    """levels (first row, size) of 8192 states or more, not the last, that hold several keys: each must read back in
    ascending order of w[W-1] << 32 | w[W-2]; returns how many there were"""
    keys = (rows[:, W - 1].astype(np.uint64) << np.uint64(32)) | (rows[:, W - 2].astype(np.uint64) if W >= 2 else 0)
    n, first = 0, 0
    for k, size in enumerate(sizes):
        lk = keys[first:first + size]
        if size >= 8192 and k + 1 < len(sizes) and len(np.unique(lk)) > 1:
            assert np.all(lk[1:] >= lk[:-1]), ("level not in key order", k, first, size)
            n += 1
        first += size
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("native", [False, "sliced"])
def test_every_row_is_its_parents_state_moved_in_one_coordinate(monkeypatch, shapes_dir, native):  # noqa: F811
    from tla_rust_b200.engine import V_RUNNING, Engine
    _clear(monkeypatch)
    monkeypatch.setenv("TLAG_SL_FORM", "scalar")       # W = 13: staged appends (sl_flush)
    s = BY_NAME["w13"]                      # 2^16 states, levels of up to 12 870: three levels the pass sorts
    cm, init, ref = _compiled(s, shapes_dir)
    e = Engine(cm, deadlock=s.stutter, native=native)
    e.seed(init)
    sizes = [len(init)]
    while True:
        ws = e.step()
        if ws["discovered"]:
            sizes.append(int(ws["discovered"]))
        if ws["verdict"] != V_RUNNING:
            break
    r = e.result()
    assert (r["distinct"], r["generated"]) == (ref.distinct, ref.generated), r
    rows = e.read_states(0, r["distinct"])
    assert _sorted_levels(rows, sizes, cm.W) >= 2, sizes
    # the box point (digit vector) of every stored row, from the reference's packed words
    where = {bytes(w): i for i, w in enumerate(np.ascontiguousarray(ref.words))}
    digit = np.array([where[bytes(w)] for w in np.ascontiguousarray(rows)])
    B = s.B + 1
    digits = np.stack([(digit // B ** i) % B for i in range(s.K)], axis=1)
    actions = set()
    for i in range(len(init), r["distinct"]):
        _, par, act, rank = e.read_link(i)
        assert 0 <= par < i and rank == 0, (i, par, rank)
        d = digits[i] - digits[par]
        assert np.count_nonzero(d) == 1 and d.sum() == 1, (i, par, digits[i], digits[par])
        actions.add(act)
    assert len(actions) == 1, actions
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("keep_going", [False, True])
def test_a_violation_that_ends_the_search_and_keep_going_match_the_oracle(monkeypatch, tmp_path, keep_going):
    from oracle import cpu_engine
    from tla_rust_b200.engine import V_RUNNING, Engine
    _clear(monkeypatch)
    s = BY_NAME["w13"]
    text, cfg = _spec(s)
    top = s.B * s.D
    text = text.replace("====", f"Inv == ~(\\A i \\in 1..8 : x[i] = {top})\n====")
    cfg += "INVARIANT Inv\n"
    path = os.path.join(str(tmp_path), f"Box_{s.name}.tla")
    with open(path, "w") as f:
        f.write(text)
    m = Model(path, cfg_text=cfg)
    st0 = m.initial_states()
    cm = compile_model(m, st0)
    init = encode_states(cm, st0)
    e = Engine(cm, deadlock=s.stutter, native=False, keep_going=keep_going)
    e.seed(init)
    last = None
    while True:
        ws = e.step()
        if ws["expanded"]:
            last = ws
        if ws["verdict"] != V_RUNNING:
            break
    r = e.result()
    assert r["verdict"] == 1, r                       # invariant violated
    if keep_going:                                    # the whole box, and the same first violation
        ref = _compiled(s, str(tmp_path / "ref"))[2]
        assert (r["generated"], r["distinct"], r["depth"]) == (ref.generated, ref.distinct, ref.depth)
        assert e.digest() == (ref.fp_xor, ref.fp_sum)
    else:
        o2 = cpu_engine.run(cm, init, n_threads=2, deadlock=s.stutter)
        assert (o2["verdict"], o2["generated"], o2["distinct"], o2["depth"]) == \
            (r["verdict"], r["generated"], r["distinct"], r["depth"]), (o2, r)
        assert last["discovered"] >= 8192, last      # the level that ends the search is one the pass would cluster
        assert e.digest() == (o2["fp_xor"], o2["fp_sum"])
    rows = e.read_states(0, r["distinct"])
    assert cpu_engine.digest(rows, cm.W) == e.digest()
    assert len(np.unique(rows, axis=0)) == r["distinct"]
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("native", ["sliced", False])
def test_reads_between_p2p_level_and_advance_level_see_every_row(monkeypatch, native):
    from oracle import cpu_engine
    from tla_rust_b200.engine import Engine
    _clear(monkeypatch)
    cm, init, exp, info = load_compiled(os.path.join(GOLDEN, "MCPaxos3_b2.tlagz"))
    o2 = cpu_engine.run(cm, init, n_threads=4, deadlock=info["deadlock"], want_states=True, max_states=1 << 22)
    lv = o2["levels"]
    e = Engine(cm, deadlock=info["deadlock"], native=native)
    e.seed(init)
    e.p2p_init(1, 0, 1 << 22)
    done, level = int(lv[0]), 1
    while lv[level]:
        first, count = e.frontier()
        ws = e.p2p_level(1, max(count, 1))
        assert ws is not None
        want = done + int(lv[level])
        assert e.result()["distinct"] == want, (level, e.result()["distinct"], want)
        x, sm, _ = o2["level_digests"][level]
        assert e.digest() == (x, sm), level          # first: tlag_digest copies the level in itself
        mid = e.read_states(0, want)
        assert cpu_engine.digest(mid, cm.W) == (x, sm), level
        e.advance_level()
        assert e.digest() == (x, sm), level
        after = e.read_states(done, want - done)
        assert np.array_equal(np.sort(after.view(np.dtype((np.void, 4 * cm.W))).ravel()),
                              np.sort(mid[done:].view(np.dtype((np.void, 4 * cm.W))).ravel())), level
        done, level = want, level + 1
    assert _sorted_levels(e.read_states(0, done), [int(n) for n in lv if n], cm.W) >= 2
    e.close()
