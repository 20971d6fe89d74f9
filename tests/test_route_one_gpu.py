"""Route mode on one GPU (-m gpu): two engines on device 0 hold ranks 0 and 1 of a partitioned search.  Each level, each
engine expands its frontier into per-owner send regions (tlag_expand_route: the route mode of the interpreter kernel,
or the route branch of the sliced kernels' successor handling), and region d of both buffers goes to engine d's
tlag_insert_records -- the host-driven exchange of DistributedBFS, with copies in place of NCCL.  Together the two
shards must hold the oracle's state set, also when a send buffer is too small and the chunk is re-run with a larger one."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from tla_rust_b200.compiled import load_compiled
from tla_rust_b200.engine import Engine, EngineError
from tla_rust_b200.fingerprint import owner_of_words

pytestmark = pytest.mark.gpu

M64 = (1 << 64) - 1


def _two_rank_bfs(name, native, cap_records):
    cm, init, exp, info = load_compiled(os.path.join(GOLDEN, name + ".tlagz"))
    W, rw = cm.W, cm.W + 2
    init = np.ascontiguousarray(init, dtype=np.uint32).reshape(-1, W)
    own = np.array([owner_of_words(w, 2, 2) for w in init])
    es = [Engine(cm, deadlock=info["deadlock"], device=0, native=native) for _ in range(2)]
    for r, e in enumerate(es):
        e.set_rank(2, r)
        e.seed(init[own == r])
    caps = [cap_records, cap_records]
    send = [torch.empty(c * rw, dtype=torch.int32, device="cuda:0") for c in caps]
    verdict, retries = 0, 0
    while True:
        counts = []
        for r, e in enumerate(es):
            _, fr = e.frontier()
            while True:
                try:
                    c, ws = e.expand_route(2, 0, fr, send[r].data_ptr(), caps[r])
                    break
                except EngineError as ex:      # send regions too small for this chunk: grow them and re-run it
                    assert "overflow" in str(ex), ex
                    caps[r] *= 2
                    retries += 1
                    send[r] = torch.empty(caps[r] * rw, dtype=torch.int32, device="cuda:0")
            counts.append(c)
            if ws["verdict"] not in (0, 5):
                verdict = ws["verdict"]
        torch.cuda.synchronize()
        for d, e in enumerate(es):
            recv = torch.cat([send[r][d * (caps[r] // 2) * rw:(d * (caps[r] // 2) + counts[r][d]) * rw] for r in range(2)])
            torch.cuda.synchronize()
            e.insert_records(recv.data_ptr(), recv.numel() // rw)
        discovered = sum(e.advance_level()["discovered"] for e in es)
        if verdict or not discovered:
            break
    rs = [e.result() for e in es]
    digests = [e.digest() for e in es]
    for e in es:
        e.close()
    return exp["o2"], dict(verdict=verdict, generated=sum(r["generated"] for r in rs), distinct=sum(r["distinct"] for r in rs),
                           depth=max(r["depth"] for r in rs), fp_xor=digests[0][0] ^ digests[1][0],
                           fp_sum=(digests[0][1] + digests[1][1]) & M64, local=[r["distinct"] for r in rs]), retries


# MCPaxos3_b2: the scalar form of the sliced kernels; MCraft: the array form
@pytest.mark.parametrize("engine", ["sliced", "interp"])
@pytest.mark.parametrize("name,cap_records", [("MCPaxos3_b2", 1 << 22), ("MCraft", 1 << 16), ("MCPaxos3_b2", 2048)])
def test_two_engines_on_one_gpu_hold_the_oracle_state_set(name, cap_records, engine):
    o2, got, retries = _two_rank_bfs(name, "sliced" if engine == "sliced" else False, cap_records)
    for k in ("verdict", "generated", "distinct", "depth", "fp_xor", "fp_sum"):
        assert got[k] == o2[k], (k, got, o2)
    assert all(0 < n < got["distinct"] for n in got["local"]), got
    if cap_records == 2048:
        assert retries >= 1                     # the send-region overflow really happened and the chunk was re-run
