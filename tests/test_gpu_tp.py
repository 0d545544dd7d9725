"""GPU (>= 2 devices): tensor-parallel shards + all-reduce reproduce the single-GPU logits
(BASELINE.json config 5).  Launches scripts/tp_check.py under torchrun; skipped on 1-GPU boxes
(runs for real on a machine with 2, 4 or 8 GPUs)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("world,shape", [(2, "512,1376,3,8,8,-1024,96"), (2, "256,688,2,8,4,512,64"),
                                         (4, "512,1376,2,8,8,-1024,64"), (8, "1024,2752,2,16,8,-2048,48")])
def test_tp_matches_single_gpu(world, shape):
    if _ngpus() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29500 + world),
           os.path.join(ROOT, "scripts", "tp_check.py"), "--shape", shape, "--steps", "20"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "PASS" in r.stdout


@pytest.mark.parametrize("n_gpus,shape", [(2, (512, 1376, 3, 8, 8, -1024, 96)), (2, (256, 688, 2, 8, 4, 512, 64)),
                                          (4, (512, 1376, 2, 8, 8, -1024, 64)), (8, (1024, 2752, 2, 16, 8, -2048, 48))])
def test_in_process_group_matches_single_gpu(n_gpus, shape):
    """SURVEY.md 8b: l2b_create(..., n_gpus) — ONE process (the Zig CLI) drives 2/4/8 GPUs through the
    same l2b_forward / l2b_forward_argmax / l2b_generate_argmax calls; logits must match the 1-GPU
    context and the oracle within 1e-4 (BASELINE.json config 5)."""
    if _ngpus() < n_gpus:
        pytest.skip(f"needs {n_gpus} GPUs")
    import numpy as np
    import llama2_zig_b200 as l2b
    import oracle_lib as O
    from llama2_zig_b200.checkpoint import shape_checkpoint
    ck = shape_checkpoint(shape)
    ck.data = l2b.synth_checkpoint_host(ck, 11)
    om = O.OracleModel(O.make_config(*ck.shape_tuple), ck.data, ck.shared_weights, W=8, kind="strict")
    with l2b.Transformer(ck, n_gpus=n_gpus) as grp, l2b.Transformer(ck) as one:
        for pos in range(min(20, ck.seq_len)):
            tok = (1 + 7919 * pos) % ck.vocab_size
            got, ref, want = grp.forward(tok, pos), one.forward(tok, pos), om.forward(tok, pos)
            scale = float(np.max(np.abs(want)))
            assert float(np.max(np.abs(got - ref))) / scale <= 1e-4, pos
            assert float(np.max(np.abs(got - want))) / scale <= 1e-4, pos
            assert grp.forward_argmax(tok, pos) == int(np.argmax(got))
        grp.reset(); one.reset()
        a = grp.generate_argmax(1, 0, 16, stop_on_bos=False)
        b = one.generate_argmax(1, 0, 16, stop_on_bos=False)
        assert a.tolist() == b.tolist()
    with l2b.Transformer(shape_checkpoint(shape), synthetic_seed=11, n_gpus=n_gpus) as syn, l2b.Transformer(ck, n_gpus=n_gpus) as grp:
        for pos in range(4):
            tok = (1 + 7919 * pos) % ck.vocab_size
            assert np.array_equal(syn.forward(tok, pos), grp.forward(tok, pos))


def test_dead_peer_returns_comm_error_instead_of_hanging():
    """ADVICE r1: the peer waits are bounded.  Rank 1 stops stepping; rank 0's next step must come
    back with L2B_ERR_COMM after L2B_SPIN_TIMEOUT_MS instead of spinning forever."""
    if _ngpus() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29533",
           os.path.join(ROOT, "scripts", "tp_check.py"), "--dead-peer"]
    env = dict(os.environ, L2B_SPIN_TIMEOUT_MS="1500")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "DEAD_PEER_OK" in r.stdout
