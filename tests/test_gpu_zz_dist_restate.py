"""The row-sharded path bit for bit (tests/dist_restate_worker.py under torchrun): the halo SpMV kernels with every
fused feature, the rank-ordered sums, the sharded Lanczos step with every orthogonalizer, project / orthogonalize, the
CG and BiCGStab steps, the block path, the dense adjoint and a replicated space against the composed restatement of
tests/dist_restate.py.  Two and three ranks always share GPU 0 (peer window only, gloo for the worker's gathers); with
at least 2 GPUs the job also runs with one rank per GPU, on the peer window and on NCCL (B2K_PEER=0).

(The file name sorts after the single-process GPU tests, like test_gpu_zz_dist.py.)"""
import os
import signal
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpus():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=30).stdout
        return sum(1 for ln in out.splitlines() if ln.startswith("GPU "))
    except (OSError, subprocess.TimeoutExpired):
        return 0


def _one_gpu():
    return {"B2K_ONE_GPU": "1", "CUDA_VISIBLE_DEVICES": os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]}


def _run(port, extra_env, nproc, timeout=600):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "dist_restate_worker.py")]
    env = dict(os.environ, **extra_env)
    # own process group: on a timeout the launcher and its workers (whose kernels may be spinning on a flag that never
    # comes) are killed together
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, cwd=ROOT, env=env,
                            start_new_session=True)
    try:
        out, err = proc.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)
        out, err = proc.communicate()
        raise AssertionError("dist_restate timed out\n" + out[-3000:] + err[-3000:])
    assert proc.returncode == 0, out[-6000:] + err[-3000:]
    assert "dist_restate ok" in out, out[-3000:]


def test_two_ranks_on_one_gpu():
    _run(29621, _one_gpu(), 2)


def test_three_ranks_on_one_gpu():
    """the middle rank has two neighbours, the shards are unequal, and an operator that couples ranks 0 and 2 is
    refused on every rank"""
    _run(29623, _one_gpu(), 3)


@pytest.mark.skipif(_ngpus() < 2, reason="needs at least 2 GPUs")
def test_one_rank_per_gpu():
    _run(29625, {}, _ngpus())


@pytest.mark.skipif(_ngpus() < 2, reason="needs at least 2 GPUs")
def test_one_rank_per_gpu_over_nccl():
    """B2K_PEER=0: halos by ncclSend/Recv and sums by ncclAllReduce; bit for bit at two ranks, bounded beyond"""
    _run(29627, {"B2K_PEER": "0"}, _ngpus())
