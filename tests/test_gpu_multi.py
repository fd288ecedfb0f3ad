"""N > 1 on real GPUs: b2a_batch_compact_* -> NCCL all-gather -> decode across ranks, checked against the
oracle on every rank.
Needs >= 2 (or 4) GPUs on one node; skipped otherwise."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.parametrize("world", [2, 4])
def test_nccl_all_gather_of_result_segments_matches_the_oracle(world):
    if _n_gpus() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29500 + world
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "workers", "nccl_shard_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    tail = "\n".join(l for l in r.stderr.splitlines() if "rank0" in l or "Error" in l or "assert" in l.lower())[-6000:]
    assert r.returncode == 0, r.stdout[-2000:] + tail
    assert f"NCCL_SHARD_OK world={world}" in r.stdout


@pytest.mark.parametrize("n_dev", [2, 4])
def test_single_process_multi_gpu_behind_the_c_abi(n_dev, oracle):
    """b2a_multi_*: one process, n devices, ncclCommInitAll + one ncclAllGather (what a Rust caller of the shim uses
    on a multi-GPU box): bit-identical to the oracle in every mode, ragged batches, a batch smaller than the device
    count, and the same results as the single-device engine."""
    if _n_gpus() < n_dev:
        pytest.skip(f"needs {n_dev} GPUs")
    import numpy as np
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from parity_util import MODES, assert_same, oracle_batch
    from rust_bio_b200 import synth
    from rust_bio_b200._lib import CScoring, MIN_SCORE
    from rust_bio_b200.engine import Engine, MultiEngine
    me = MultiEngine(list(range(n_dev)))
    assert me.n_devices == n_dev
    print("exchange:", me.exchange_kind)
    cs = CScoring(-5, -1, MIN_SCORE, MIN_SCORE, MIN_SCORE, MIN_SCORE, 1, -1, 1, None, None, 0)
    s, _ = oracle.make_scoring(-5, -1, 1, -1)
    single = Engine(0)
    try:
        for mode, batch in (("local", synth.uniform_pairs(synth.BASES["C1"], 0, 5001, 150, 150)),
                            ("global", synth.ragged_pairs(9, 1203, 260, 300)),
                            ("semiglobal", synth.ragged_pairs(10, n_dev - 1, 60, 90))):
            ref, ref_ops = oracle_batch(oracle, mode, s, batch, threads=8)
            for rep in range(2):
                res = me.align_batch(MODES[mode], cs, batch)
                n = len(batch[2])
                assert_same(res.as_dict(), [res.ops_of(i) for i in range(n)], ref, ref_ops, batch, f"multi {n_dev} {mode}")
            one = single.align_batch(MODES[mode], cs, batch)
            tot = int(one.ops_off[n])
            assert np.array_equal(one.ops[:tot], res.ops[:tot]) and np.array_equal(one.clip_len, res.clip_len)
        assert int(me.stats.cells) > 0
    finally:
        single.close()
        me.close()
