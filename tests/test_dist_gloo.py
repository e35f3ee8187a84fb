"""World-size-2 ``gloo`` test (CPU) of the data-parallel host logic in dynaboa_b200/dist.py: frame sharding,
the outer-gradient all-reduce(mean) hook, the rank-consistent dynamic-loop decision and max-over-ranks timing."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    from dynaboa_b200 import dist as dd
    r, w, _ = dd.init_from_env(backend='gloo')
    assert (r, w) == (rank, world)
    # 1. gradient all-reduce hook: every rank ends with the mean of the per-rank flat gradients
    g = torch.Generator().manual_seed(100 + rank)
    grad = torch.randn(10007, generator=g)
    mine = grad.clone()
    dd.make_grad_sync(world)(grad)
    others = [torch.randn(10007, generator=torch.Generator().manual_seed(100 + k)) for k in range(world)]
    assert torch.allclose(grad, sum(others) / world, atol=1e-6)
    # 2. dynamic-loop decision: summed (a.b, |a|^2, |b|^2) reproduce the whole-batch cosine on every rank
    feats_a = [torch.randn(1, 1024, generator=torch.Generator().manual_seed(200 + k)) for k in range(world)]
    feats_b = [a + 0.01 * torch.randn(1, 1024, generator=torch.Generator().manual_seed(300 + k)) for k, a in enumerate(feats_a)]
    a, b = feats_a[rank].double(), feats_b[rank].double()
    cos = dd.allreduce_cosine_terms((a * b).sum(), (a * a).sum(), (b * b).sum())
    ref = F.cosine_similarity(torch.cat(feats_a).flatten().double(), torch.cat(feats_b).flatten().double(), dim=0)
    assert abs(float(cos) - float(ref)) < 1e-12
    # 3. timing is reported as the max over ranks
    assert dd.max_over_ranks(1.0 + rank) == float(world)
    out[rank] = (dd.shard_range(11, rank, world), float(mine.sum()))
    dist.destroy_process_group()


def test_world_size_2_gloo():
    world, port = 2, _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    shards = [out[r][0] for r in range(world)]
    assert shards == [(0, 6), (6, 11)]                      # contiguous, covering, first ranks take the remainder


def test_gradient_buckets_partition_the_arena_into_whole_layers():
    """The three spans ``BucketedGradSync`` all-reduces partition [0, arena_floats) and each holds whole parameters of the layers
    whose gradients the backward has finished when it records that bucket's event: layer4 and the head (bucket 0), layer3
    (bucket 1), then the stem, layer1 and layer2 (bucket 2)."""
    from harness import built_lib
    from dynaboa_b200.hmr import ArenaLayout
    lib = built_lib()
    lay = ArenaLayout()
    bounds = [(lib.dboa_hmr_bucket_offset(k), lib.dboa_hmr_bucket_offset(k - 1)) for k in range(3)]
    assert bounds[0][1] == lay.floats and bounds[2][0] == 0
    assert all(lo < hi for lo, hi in bounds) and bounds[0][0] == bounds[1][1] and bounds[1][0] == bounds[2][1]
    first = dict(zip(lay.names, lay.offsets))
    assert bounds[0][0] == first['layer4.0.conv1.weight'] and bounds[1][0] == first['layer3.0.conv1.weight']
    owner = lambda name: 0 if name.split('.')[0] in ('layer4', 'fc1', 'fc2', 'decpose', 'decshape', 'deccam') else (
        1 if name.startswith('layer3.') else 2)
    for name, off, shape, stride in zip(lay.names, lay.offsets, lay.shapes, lay.strides):
        end = off + 1 + sum((s - 1) * st for s, st in zip(shape, stride))
        lo, hi = bounds[owner(name)]
        assert lo <= off and end <= hi, (name, off, end, owner(name), bounds)


def test_shard_range_partitions():
    from dynaboa_b200.dist import shard_range
    for n in (0, 1, 7, 8, 64):
        for w in (1, 2, 4, 8):
            spans = [shard_range(n, r, w) for r in range(w)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            assert max(h - l for l, h in spans) - min(h - l for l, h in spans) <= 1
