"""bench.py contract pieces that need no GPU: the reference arm's JSON line on the small workload (run for real on the host cores: the unmodified
reference from oracle/_ref where it was installed, else the oracle port), rank != 0 of a multi-rank reference launch doing nothing, the workload
tables, and the arrays --dump-outputs writes."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, env=None, timeout=900):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True, timeout=timeout, env=e, cwd=ROOT)


def test_reference_arm_line_small_workload():
    r = _run(["--impl", "reference", "--workload", "conformer_4l256_joint_8x5s", "--steps", "2", "--warmup", "1"])
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    assert line["impl"] == "reference" and line["unit"] == "utterances/s" and line["higher_is_better"] is True and line["value"] > 0
    assert line["steps"] == 2 and line["config"]["workload"] == "conformer_4l256_joint_8x5s" and line["gpu_launches"] == 0
    cb = line["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and cb["value"] == line["value"] and "sample" in cb
    assert line["e2e"] == {"value": line["value"], "unit": "utterances/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_reference_arm_other_ranks_exit_without_work():
    r = _run(["--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "0"], env={"RANK": "1", "LOCAL_RANK": "1", "WORLD_SIZE": "2"}, timeout=120)
    assert r.returncode == 0 and not [ln for ln in r.stdout.splitlines() if ln.startswith("{")]


def test_workload_tables():
    sys.path.insert(0, ROOT)
    import bench

    assert set(bench.LM_FUSION) <= set(bench.WORKLOADS) and not (set(bench.STREAMING) & set(bench.WORKLOADS))
    for name, (cfg, secs, batch, beam, ctcw, mlr) in bench.WORKLOADS.items():
        assert cfg["d_model"] % cfg["heads"] == 0 and secs > 0 and batch > 0 and 0 < beam <= 64 and 0.0 <= ctcw <= 1.0 and mlr < 0, name


def test_dump_outputs_writes_float_arrays(tmp_path):
    """--dump-outputs: best hypothesis per utterance as float64 arrays (token ids padded with -1), one .npy per name."""
    import numpy as np
    import torch

    sys.path.insert(0, ROOT)
    import bench
    from espnet_b200.search import Hypothesis

    res = [[Hypothesis(yseq=torch.tensor([4, 7, 9, 4]), score=-1.5, scores={"decoder": -1.0, "ctc": -2.0})], [],
           [Hypothesis(yseq=torch.tensor([4, 4]), score=-0.25, scores={"decoder": -0.5, "ctc": 0.0})]]
    bench.dump_outputs(str(tmp_path / "d"), bench.hyps_arrays(res))
    tok = np.load(tmp_path / "d" / "tokens.npy")
    assert tok.dtype == np.float64 and tok.tolist() == [[4, 7, 9, 4], [-1, -1, -1, -1], [4, 4, -1, -1]]
    assert np.load(tmp_path / "d" / "lengths.npy").tolist() == [4, 0, 2]
    sc = np.load(tmp_path / "d" / "score.npy")
    assert sc[0] == -1.5 and np.isnan(sc[1]) and sc[2] == -0.25
    assert np.load(tmp_path / "d" / "score_ctc.npy")[2] == 0.0


def test_dump_outputs_refused_where_it_records_nothing():
    for args in (["--impl", "reference", "--dump-outputs", "d"], ["--steps", "0", "--dump-outputs", "d"]):
        r = _run(args, timeout=120)
        assert r.returncode == 2 and "--dump-outputs" in r.stderr, r.stderr[-500:]


def _gather_worker(rank, world, port, q):
    import numpy as np
    import torch.distributed as dist

    sys.path.insert(0, ROOT)
    import bench

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    toks = [[1, 2, 3]] if rank == 0 else [[7], [8, 9, 10, 11]]
    out = bench.gather_arrays(bench.tokens_arrays(toks), world)
    if rank == 0:
        q.put({k: np.asarray(v).tolist() for k, v in out.items()})
    dist.destroy_process_group()


def test_dump_outputs_gathers_every_rank_in_rank_order():
    """With several ranks the dump holds every rank's streams / utterances, rank 0 first, padded to the widest shard."""
    import socket

    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
    assert out["tokens"] == [[1, 2, 3, -1], [7, -1, -1, -1], [8, 9, 10, 11]]
    assert out["lengths"] == [3, 1, 4]
