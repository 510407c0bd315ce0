"""CPU test of the N > 1 host path (gloo, world_size 2): frame-pair sharding, the broadcast of the
NCCL unique id over torch.distributed, and the agreement on the all-gather slot size."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_world_size_2_gloo(tmp_path):
    pairs = 29
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "_rank_worker.py"), str(pairs), str(tmp_path)]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env)
    assert res.returncode == 0, res.stderr[-2000:]
    outs = [json.load(open(tmp_path / ("rank%d.json" % r))) for r in range(2)]
    covered = []
    for o in outs:
        covered += list(range(o["lo"], o["hi"]))
    assert covered == list(range(pairs))
    expect = (np.arange(128) * 7 + 3).astype(np.uint8)
    assert all(o["id_sum"] == int(expect.sum()) and o["id0"] == int(expect[1]) for o in outs)
    want_slot = ((1000 + 777 + 7) // 8 + 15) // 16 * 16
    assert all(o["slot"] == want_slot for o in outs)
    # strong-scaling layout (ShardedStreamEncoder's host logic): equal slot counts, one halo frame, stream-ordered rows
    for o in outs:
        lay = o["layout"]
        assert lay["slots"] == 15 and lay["frames"] == lay["pairs"] + 1 and lay["first_frame"] == lay["lo"] == o["lo"]
        assert [h[0] for h in o["headers"]] == list(range(pairs))
        assert [tuple(r) for r in o["rows"]] == [(h[1], h[0] - outs[h[1]]["lo"]) for h in o["headers"]]


class _NoCollectives:
    """A rank of `world` whose collectives must not be reached."""

    def __init__(self, rank, world):
        self.rank, self.world = rank, world

    def get_rank(self):
        return self.rank

    def get_world_size(self):
        return self.world

    def __getattr__(self, name):
        raise AssertionError("collective %s entered" % name)


def test_sharded_encoder_needs_a_pair_per_rank():
    """Fewer frame pairs than ranks: every rank, including those that would own a pair, raises ValueError in the constructor,
    before any collective and before the library is touched (so this runs without a GPU)."""
    from new_bloom_filter_repo_b200 import distributed as rdist
    for world, total_frames in ((4, 3), (2, 2), (3, 1), (1, 1), (16, 16)):
        for rank in range(world):
            with pytest.raises(ValueError, match="every rank needs at least one pair"):
                rdist.ShardedStreamEncoder(_NoCollectives(rank, world), 8, 8, 3, np.uint8, total_frames, max_l_bits=64)
