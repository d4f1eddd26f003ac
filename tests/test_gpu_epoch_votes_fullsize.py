"""The vote form at full size (2^20 validators, 2 048 committees of 512, bench.build_world's world): 2 votes per committee at 95 %
participation.  Exactly the planted corrupt votes are rejected, and the aggregate signature of a sample of votes equals Sign(sum of the
attesters' secret keys, the vote's message) by linearity (sk_i = sk0 + i * delta), as test_gpu_fullsize.py checks per committee."""
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
NONE = 0xFFFFFFFF


def test_full_size_split_epoch():
    import bench
    from pos_evolution_b200 import spec as PS
    from pos_evolution_b200.engine import Engine
    from pos_evolution_b200.epoch import EpochProcessor
    eng = Engine(0)
    W = bench.build_world(eng, 0, np, PS)
    A, C, N = bench.N_AGG, bench.COMMITTEE_SIZE, bench.N_VAL
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(12)
    com = np.repeat(np.arange(A, dtype=np.int64), C)
    vote = com * 2 + rng.integers(0, 2, size=N)
    msgs = np.frombuffer(b"".join(hashlib.sha256(b"full/vote%d" % v).digest() for v in range(2 * A)), dtype=np.uint8).reshape(-1, 32)
    sk = [W["sk0"] + i * W["delta"] for i in range(N)]
    sk8 = np.frombuffer(b"".join(k.to_bytes(32, "little") for k in sk), dtype=np.uint32).reshape(N, 8)
    sigs = eng.sign(np.ascontiguousarray(sk8[W["members"]]), vote.astype(np.uint32), msgs)
    vote = np.where(rng.random(N) < 0.95, vote, NONE)
    # corrupt votes: one attester's signature over another vote's message
    bad = sorted(rng.choice(2 * A, size=6, replace=False).tolist())
    for v in bad:
        j = int(np.nonzero(vote == v)[0][0])
        sigs[j] = eng.sign(sk8[W["members"][j]:W["members"][j] + 1], [0], msgs[(v + 2) % (2 * A):(v + 2) % (2 * A) + 1])[0]
    vote_off = np.arange(A + 1, dtype=np.int64) * 2
    ep = EpochProcessor(eng, A, N, C // 8, bench.N_BLOCKS, device=dev, depth=3, max_votes=2 * A)
    ep.set_committees(W["members"], W["off"])
    d = [torch.as_tensor(sigs, device=dev), None, torch.as_tensor(msgs, device=dev), torch.full((2 * A,), 5, dtype=torch.int64, device=dev),
         torch.as_tensor((bench.N_BLOCKS - 1 - (np.arange(2 * A) % 64)).astype(np.int32), device=dev)]
    ok, head = ep.process_epoch_dev(*d, 0, bench.N_BLOCKS - 1, W["boost"],
                                    votes=(torch.as_tensor(vote.astype(np.uint32).view(np.int32), device=dev), vote_off))
    torch.cuda.synchronize()
    assert eng.guard_flags() == 0
    expect = np.ones(2 * A, dtype=np.uint8)
    expect[bad] = 0
    assert np.array_equal(ok.cpu().numpy(), expect)
    agg = ep.slots[0].agg_sig[:2 * A].cpu().numpy()
    rows = ep.slots[0].v_aggbits[:2 * A].cpu().numpy()
    R = bench.R_ORDER
    for v in rng.choice([v for v in range(2 * A) if v not in bad], size=12, replace=False).tolist():
        c = v // 2
        att = [int(W["members"][c * C + j]) for j in range(C) if vote[c * C + j] == v]
        assert [j for j in range(C) if (rows[v, j >> 3] >> (j & 7)) & 1] == [j for j in range(C) if vote[c * C + j] == v]
        want = eng.sign([sum(sk[x] for x in att) % R], [0], msgs[v:v + 1])[0]
        assert bytes(agg[v]) == bytes(want), v
    eng.close()
