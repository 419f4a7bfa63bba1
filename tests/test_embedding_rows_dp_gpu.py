"""On one GPU: the data-parallel gradient scatter (lb_embed_rows_scatter_dp) with W = 2 and 4 ranks
simulated on one device -- W id buffers, one row-state copy per simulated rank, no handshake -- against
one world = 1 scatter of the concatenated batch and a float64 oracle; plus the flag handshake with
the peers' flags already published."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
V, D, S = 1000, 48, 77


def _state(table, cap, placeholders, decay=1.0):
    st = {"slot_of": torch.full((V,), -1, device=DEV, dtype=torch.int32),
          "slot_tok": torch.full((cap,), -1, device=DEV, dtype=torch.int32),
          "state": torch.zeros(4, device=DEV, dtype=torch.int32),
          "decay": torch.full((1,), decay, device=DEV, dtype=torch.float64),
          "master": torch.zeros(cap, D, device=DEV), "grad": torch.zeros(cap, D, device=DEV)}
    idx = torch.tensor(placeholders, device=DEV)
    st["slot_of"][idx] = torch.arange(len(placeholders), device=DEV, dtype=torch.int32)
    st["slot_tok"][: len(placeholders)] = idx.to(torch.int32)
    st["master"][: len(placeholders)] = table[idx].float()
    st["state"][:2] = len(placeholders)
    return st


def _rest(st, table, cap):
    from lora_b200._C import dtype_code, ptr
    return (ptr(st["slot_of"]), ptr(st["slot_tok"]), cap, ptr(st["state"]), ptr(table), dtype_code(table.dtype),
            ptr(st["decay"]), ptr(st["master"]), ptr(st["grad"]))


def _scatter_dp(ids_list, rank, grad, st, table, cap, flags=None, epoch=None):
    from lora_b200._C import check, dtype_code, lib, ptr, stream_ptr
    w = len(ids_list)
    ids_p = (ctypes.c_void_p * w)(*[t.data_ptr() for t in ids_list])
    fl = None if flags is None else (ctypes.c_void_p * w)(*[f.data_ptr() for f in flags])
    check(lib.lb_embed_rows_scatter_dp(ids_p, w, rank, ids_list[0].numel(), ptr(grad), dtype_code(grad.dtype), D, V,
                                       *_rest(st, table, cap), fl, ptr(epoch), stream_ptr()),
          "lb_embed_rows_scatter_dp")


def _scatter_one(ids, grad, st, table, cap):
    from lora_b200._C import check, dtype_code, lib, ptr, stream_ptr
    check(lib.lb_embed_rows_scatter(ptr(ids), ptr(grad), dtype_code(grad.dtype), ids.numel(), D, V,
                                    *_rest(st, table, cap), stream_ptr()), "lb_embed_rows_scatter")


def _commit(st):
    """What the write-back and the optimizer launch leave for the next scatter: claims committed,
    slot gradients zeroed."""
    st["state"][0] = st["state"][1]
    st["grad"].zero_()


def _batch(W, B, g, pool):
    ids = [pool[torch.randint(0, pool.numel(), (B * S,), device=DEV, generator=g)].contiguous() for _ in range(W)]
    return ids


KEYS = ("slot_of", "slot_tok", "state", "master")


@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
def test_ranks_agree_and_sum_to_the_concatenated_batch(W, gdtype):
    torch.manual_seed(0)
    g = torch.Generator(device=DEV).manual_seed(W)
    table = torch.randn(V, D, device=DEV).to(torch.bfloat16)
    cap, B, ph, dk = 256, 2, [998, 999], 0.97
    ranks = [_state(table, cap, ph, dk) for _ in range(W)]
    one = _state(table, cap, ph, dk)
    seen = set(ph)
    for step in range(2):                        # the second step starts from committed claims
        pool = torch.arange(40 * step, 40 * step + 60, device=DEV)
        ids = _batch(W, B, g, pool)
        ids[0][3] = 998
        only_last = 900 + step                   # occurs on the last rank only
        ids[W - 1][5] = only_last
        grads = [torch.randn(B * S, D, device=DEV, generator=g).to(gdtype) for _ in range(W)]
        for r in range(W):
            _scatter_dp(ids, r, grads[r], ranks[r], table, cap)
        cat_ids, cat_g = torch.cat(ids), torch.cat(grads)
        _scatter_one(cat_ids, cat_g, one, table, cap)
        torch.cuda.synchronize()
        for r in range(1, W):                    # every replica holds the same claims, bit for bit
            for k in KEYS:
                assert torch.equal(ranks[r][k], ranks[0][k]), (r, k)
        for k in KEYS:                           # ... and they are those of one process on the whole batch
            assert torch.equal(ranks[0][k], one[k]), k
        n = int(one["state"][1])
        toks = one["slot_tok"][:n].long()
        seen |= set(cat_ids.tolist())
        assert set(toks.tolist()) == seen
        dense = torch.zeros(V, D, dtype=torch.float64, device=DEV)
        dense.index_add_(0, cat_ids, cat_g.double())
        summed = sum(st["grad"][:n].double() for st in ranks)
        assert float((summed - dense[toks]).norm() / dense[toks].norm()) < 1e-6
        assert float((one["grad"][:n].double() - dense[toks]).norm() / dense[toks].norm()) < 1e-6
        # a token of the last rank only: claimed everywhere from the decayed stored row, no local gradient
        s = int(ranks[0]["slot_of"][only_last])
        assert s >= len(ph)
        want = (table[only_last].double() * dk).float()
        for r in range(W - 1):
            assert torch.equal(ranks[r]["master"][s], want), r
            assert int(ranks[r]["grad"][s].count_nonzero()) == 0, r
        assert int(ranks[W - 1]["grad"][s].count_nonzero()) > 0
        for st in ranks + [one]:
            _commit(st)
    assert all(int(st["state"][3]) == 0 for st in ranks)


@pytest.mark.parametrize("W", [2, 4])
def test_union_overflow_is_flagged_on_every_rank(W):
    table = torch.randn(V, D, device=DEV)
    cap = 24
    ranks = [_state(table, cap, [999]) for _ in range(W)]
    # 12 distinct tokens per rank (fits alone: 1 + 12 <= 24), 12 * W over all ranks (does not)
    ids = [torch.arange(100 + 12 * r, 112 + 12 * r, device=DEV).repeat(7)[:S].contiguous() for r in range(W)]
    for r in range(W):
        alone = _state(table, cap, [999])
        _scatter_dp(ids[r:r + 1], 0, torch.randn(S, D, device=DEV), alone, table, cap)
        torch.cuda.synchronize()
        assert int(alone["state"][3]) == 0
    for r in range(W):
        _scatter_dp(ids, r, torch.randn(S, D, device=DEV), ranks[r], table, cap)
    torch.cuda.synchronize()
    for r in range(W):
        assert int(ranks[r]["state"][3]) & 1, r
        assert int(ranks[r]["state"][1]) == cap
        for k in KEYS:
            assert torch.equal(ranks[r][k], ranks[0][k]), (r, k)


@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
def test_world_one_is_bitwise_the_single_process_scatter(gdtype):
    g = torch.Generator(device=DEV).manual_seed(5)
    table = torch.randn(V, D, device=DEV)
    cap = 128
    a, b = _state(table, cap, [997], 0.9), _state(table, cap, [997], 0.9)
    ids = torch.randint(0, 50, (2 * S,), device=DEV, generator=g)
    grad = torch.randn(2 * S, D, device=DEV, generator=g).to(gdtype)
    _scatter_dp([ids], 0, grad, a, table, cap)
    _scatter_one(ids, grad, b, table, cap)
    torch.cuda.synchronize()
    for k in KEYS + ("grad", "decay"):
        assert torch.equal(a[k], b[k]), k


def test_handshake_publishes_the_epoch_and_reads_published_peers():
    """Rank 0 of 3 with the handshake on; the simulated peers' flags are already at the epoch, so the
    launch never waits. It must publish its epoch, advance its counter once per launch and compute
    what the launch without a handshake computes."""
    g = torch.Generator(device=DEV).manual_seed(6)
    table = torch.randn(V, D, device=DEV)
    cap, W = 256, 3
    ids = [torch.randint(0, 300, (S,), device=DEV, generator=g) for _ in range(W)]
    grad = torch.randn(S, D, device=DEV, generator=g)
    flags = [torch.zeros(1, device=DEV, dtype=torch.int32) for _ in range(W)]
    epoch = torch.zeros(2, device=DEV, dtype=torch.int32)
    for e in (1, 2):
        for f in flags[1:]:
            f.fill_(e)
        with_hs, without = _state(table, cap, [999]), _state(table, cap, [999])
        _scatter_dp(ids, 0, grad, with_hs, table, cap, flags=flags, epoch=epoch)
        _scatter_dp(ids, 0, grad, without, table, cap)
        torch.cuda.synchronize()
        assert int(flags[0]) == e and epoch.tolist() == [e, 0]
        for k in KEYS + ("grad",):
            assert torch.equal(with_hs[k], without[k]), k
