"""The cross-partition exchange plan (calfkit/engine/exchange.py: plan_exchange) against a plain loop over the
publish table, for every rank of several world sizes.  plan_exchange is the tensor statement the device plan
kernels (ck_exchange_plan, and the ck_xplan_* kernels of ck_exchange_send) are pinned to on the GPU."""
import numpy as np
import pytest
import torch

from calfkit.engine.exchange import plan_exchange


def _table(seed: int):
    """a publish table (payload, topic_id, topic_off, topic_len, record, has_key, partition, pad) with keyed, unkeyed
    and empty slots; several publishes may share a payload, as a fan-out's do"""
    rng = np.random.default_rng(seed)
    npay, npubs = 120, 400
    lens = rng.integers(0, 300, size=npay)
    out_off = np.concatenate([[0], np.cumsum((lens + 15) & ~15)]).astype(np.int64)      # 16-byte aligned starts
    pubs = np.zeros((npubs, 8), dtype=np.int32)
    pubs[:, 0] = rng.integers(0, npay, size=npubs)
    pubs[:, 1] = rng.integers(0, 5, size=npubs)
    pubs[:, 4] = rng.integers(0, 200, size=npubs)
    kind = rng.integers(0, 4, size=npubs)          # 0, 1: keyed  2: unkeyed  3: no publish in this slot
    pubs[:, 5] = kind <= 1
    pubs[:, 6] = np.where(kind <= 1, rng.integers(0, 2**31 - 1, size=npubs, dtype=np.int64), -1)
    pubs[kind == 3, 0] = -1
    pubs[:4, 6] = [0, 1, 2**31 - 1, 7]             # extreme partitions
    pubs[:4, 5] = 1
    pubs[4, 5], pubs[4, 6], pubs[4, 0] = 1, 5, -1  # keyed but without a payload: never forwarded
    return pubs, out_off, lens.astype(np.int32)


def _expect(pubs, out_off, lens, rank: int, world: int):
    """what a rank forwards: the keyed publishes owned by another rank, grouped by destination in table order"""
    sel = []
    for d in range(world):
        if d == rank:
            continue
        for i in range(len(pubs)):
            if pubs[i, 5] == 1 and pubs[i, 0] != -1 and int(pubs[i, 6]) % world == d:
                sel.append(i)
    counts, nbytes = [0] * world, [0] * world
    src_off, ln, dst_off, pos = [], [], [], 0
    for i in sel:
        p = int(pubs[i, 0])
        d = int(pubs[i, 6]) % world
        counts[d] += 1
        nbytes[d] += int(lens[p])
        src_off.append(int(out_off[p]))
        ln.append(int(lens[p]))
        dst_off.append(pos)
        pos += int(lens[p])
    return sel, counts, nbytes, src_off, ln, dst_off


@pytest.mark.parametrize("world,rank", [(w, r) for w in (1, 2, 3, 8) for r in range(w)])
def test_plan_exchange_matches_loop(world, rank):
    pubs, out_off, lens = _table(seed=31 * world + rank)
    plan = plan_exchange(torch.from_numpy(pubs), torch.from_numpy(out_off), torch.from_numpy(lens), rank, world)
    sel, counts, nbytes, src_off, ln, dst_off = _expect(pubs, out_off, lens, rank, world)
    if world > 1:
        assert sel, "the table should forward something"
    assert plan.sel.tolist() == sel
    assert plan.counts.tolist() == counts
    assert plan.nbytes.tolist() == nbytes
    assert plan.src_off.tolist() == src_off
    assert plan.lens.tolist() == ln
    assert plan.dst_off.tolist() == dst_off
