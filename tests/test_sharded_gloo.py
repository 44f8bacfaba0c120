"""Host logic of the multi-GPU forward (esac_b200/sharded.py) on CPU: world_size-2 gloo, fake local pipelines."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from esac_b200 import sharded


def test_select_global_is_first_strict_maximum():
    M = 5
    g = np.zeros((3, M + 21))
    g[0, :M] = [1, 2, 3, 2, 1]
    g[1, :M] = [3, 9, 9, 0, 0]       # tie inside rank 1: the first one wins
    g[2, :M] = [9, 0, 0, 0, 0]       # tie across ranks: the lower global index wins
    for r in range(3):
        g[r, M:M + 16] = np.eye(4).reshape(-1) * (r + 1)
        g[r, M + 16] = 10 + r
        g[r, M + 18:M + 21] = [M, r * M, 1]   # M, hyp_offset, hyp_stride
    w, rank, pose, expert, probs = sharded.select_global(g, M)
    assert (w, rank, expert) == (6, 1, 11)
    assert pose[0, 0] == 2.0 and abs(probs.sum() - 1) < 1e-12


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q, unequal=False):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    M = (9 if rank == 1 else 0) if unequal else 6   # unequal: rank 0 holds NO hypotheses, rank 1 nine
    rng = np.random.default_rng(rank)
    scores = torch.from_numpy(rng.uniform(0, 50, M))
    if rank == 1:
        scores[4] = 77.0  # the global winner lives on rank 1

    def fake_local(coords, assign, params):
        lw = int(torch.argmax(scores))
        pose = torch.eye(4) * (rank + 1)
        return scores, pose, 2, lw  # local expert id 2

    out = torch.zeros(4, 4)
    e = sharded.forward_sharded(torch.zeros(3, 3, 2, 2), torch.zeros(M, dtype=torch.int64), out, (), expert_offset=rank * 3,
                                local_forward=fake_local)
    q.put((rank, e, out.numpy().copy().tolist()))
    dist.barrier()
    dist.destroy_process_group()


def test_forward_sharded_world2_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    for p in ps:
        p.join(timeout=240)
        assert p.exitcode == 0
    res = [q.get(timeout=5) for _ in range(2)]
    for rank, e, pose in res:
        assert e == 1 * 3 + 2          # rank 1's shard, local expert 2
        assert np.allclose(pose, np.eye(4) * 2)


def test_forward_sharded_unequal_and_empty_shards_gloo():
    """Real gating draws give every expert shard a different hypothesis count, possibly zero: records are padded to the
    largest shard with -inf scores and an empty shard contributes an all -inf record."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q, True)) for r in range(2)]
    for p in ps:
        p.start()
    for p in ps:
        p.join(timeout=240)
        assert p.exitcode == 0
    for rank, e, pose in [q.get(timeout=5) for _ in range(2)]:
        assert e == 1 * 3 + 2
        assert np.allclose(pose, np.eye(4) * 2)


def test_select_global_ignores_padding():
    M_pad = 4
    g = np.full((2, M_pad + 21), -1.0)
    g[0, :M_pad] = [5.0, -np.inf, -np.inf, -np.inf]      # rank 0 holds one hypothesis
    g[1, :M_pad] = [1.0, 9.0, 9.0, 2.0]
    g[1, M_pad:M_pad + 16] = np.eye(4).reshape(-1) * 3
    g[1, M_pad + 16] = 7
    g[0, M_pad + 18:M_pad + 21] = [1, 0, 1]
    g[1, M_pad + 18:M_pad + 21] = [4, 1, 1]
    w, rank, pose, expert, probs = sharded.select_global(g, M_pad)
    assert (w, rank, expert) == (M_pad + 1, 1, 7) and pose[0, 0] == 3.0
    assert probs[1] == 0.0 and abs(probs.sum() - 1) < 1e-12


def _exchange_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ex = sharded.make_exchange()
    scores = np.array([[3.0, 7.0, 1.0], [9.0, 2.0, 8.5]])[rank]
    mx = scores.max()
    g = ex(1, [mx, np.exp(scores - mx).sum()])
    tot = ex(2, [float(rank + 1) * 0.25])
    q.put((rank, g, tot))
    dist.barrier()
    dist.destroy_process_group()


def test_backward_exchange_world2_gloo():
    """The two reductions of the sharded backward (global softmax normalisation, global expected loss)."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_exchange_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    for p in ps:
        p.join(timeout=240)
        assert p.exitcode == 0
    allsc = np.array([3.0, 7.0, 1.0, 9.0, 2.0, 8.5])
    for _ in range(2):
        rank, g, tot = q.get(timeout=5)
        assert abs(g[0] - 9.0) < 1e-15 and abs(g[1] - np.exp(allsc - 9.0).sum()) < 1e-12
        assert abs(tot[0] - 0.75) < 1e-15


def test_select_global_breaks_ties_in_the_unsharded_order_with_strided_shards():
    """Hypotheses dealt round-robin (hyp_stride = world): a tie between global hypotheses 3 (rank 1, local 1) and 4 (rank 0,
    local 2) goes to hypothesis 3 although rank 0 comes first in the gathered buffer."""
    M_pad = 3
    g = np.full((2, M_pad + 21), -1.0)
    g[0, :M_pad] = [1.0, 2.0, 8.0]     # global 0, 2, 4
    g[1, :M_pad] = [0.0, 8.0, 3.0]     # global 1, 3, 5
    for r in range(2):
        g[r, M_pad:M_pad + 16] = np.eye(4).reshape(-1) * (r + 1)
        g[r, M_pad + 16] = r
        g[r, M_pad + 18:M_pad + 21] = [3, r, 2]
    w, rank, pose, expert, _ = sharded.select_global(g, M_pad)
    assert (w, rank, expert) == (M_pad + 1, 1, 1) and pose[0, 0] == 2.0


def test_forward_sharded_refuses_a_call_in_which_no_shard_holds_a_hypothesis(tmp_path):
    """esac.forward refuses M = 0, and so does the sharded forward when every rank's hypAssignment is empty: the torch route
    with the library's message (one-rank gloo group in this process)."""
    def never(coords, assign, params):
        raise AssertionError("a shard without hypotheses runs no local pipeline")

    dist.init_process_group("gloo", store=dist.FileStore(str(tmp_path / "store"), 1), rank=0, world_size=1)
    try:
        with pytest.raises(RuntimeError, match="no shard holds a hypothesis"):
            sharded.forward_sharded(torch.zeros(1, 3, 2, 2), torch.zeros(0, dtype=torch.int64), torch.zeros(4, 4), (),
                                    expert_offset=0, local_forward=never, M_pad=4)
    finally:
        dist.destroy_process_group()
