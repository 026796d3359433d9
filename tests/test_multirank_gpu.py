"""The multi-rank path against the oracle (SURVEY.md 8(a) row a10: treeAggregate's cross-partition reduce,
AGD.scala:196-204, replaced by P2P stores + epoch flags into peer HBM, csrc/xchg.cu).

One PROCESS per rank, as under torchrun / one Spark executor per GPU.  On a box with a single GPU both ranks share
device 0: the exchange buffers are then mapped through CUDA IPC on the same device and the handles travel through the
host (transport="ipc", no NCCL -- NCCL refuses two ranks on one GPU), so the IPC + epoch-flag protocol is exercised
even where only one GPU exists.  With two or more GPUs the same worlds also run one rank per GPU over both transports."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from k1_reference import bf16_to_f32, f32_to_bf16_bits, row_selected, row_terms  # noqa: E402
from mp_worker import MB_FRACTION, MB_ITERS, make_csr, make_data, minibatch_poisoned  # noqa: E402


def _gpu_count():
    try:
        import ctypes
        cuda = ctypes.CDLL("libcuda.so.1")
        if cuda.cuInit(0) != 0:
            return 0
        n = ctypes.c_int()
        return n.value if cuda.cuDeviceGetCount(ctypes.byref(n)) == 0 else 0
    except OSError:
        return 0


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _spawn_world(world, devices, transport, out, timeout=420):
    port = _free_port()
    env = dict(os.environ, OMP_NUM_THREADS="1")
    procs = [subprocess.Popen([sys.executable, os.path.join(HERE, "mp_worker.py"), str(r), str(world), str(port),
                               str(devices[r]), transport, out], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
             for r in range(world)]
    logs, failed = [], False
    for p in procs:
        try:
            o, _ = p.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            failed = True
            for q in procs:          # exactly the PIDs this test started
                q.kill()
            o, _ = p.communicate()
        logs.append(o.decode(errors="replace")[-3000:])
        failed = failed or p.returncode != 0
    assert not failed, "a rank failed or hung:\n" + "\n-----\n".join(logs)
    with open(out) as f:
        return json.load(f)


WORLDS = [("ipc", 2, "same"), ("ipc", 3, "same"), ("ipc", 2, "spread"), ("nccl", 2, "spread")]


@pytest.mark.gpu
@pytest.mark.parametrize("transport,world,placement", WORLDS)
def test_process_per_rank_world_matches_oracle(oracle, tmp_path, transport, world, placement):
    ngpu = _gpu_count()
    if placement == "spread" and ngpu < world:
        pytest.skip(f"needs {world} GPUs (the same-device worlds cover the IPC path on this box)")
    devices = list(range(world)) if placement == "spread" else [0] * world
    res = _spawn_world(world, devices, transport, str(tmp_path / "res.json"))
    O = oracle
    # --- applySmooth and the loop on loaded shards, oracle partitions = ranks (the same combOp order, AGD.scala:201-204)
    X, y = make_data(6001, 1024, 7)
    w = np.random.default_rng(11).standard_normal(1024) * 0.1
    D = O.Data(y, X=X)
    loss, g, cnt = O.smooth(D, "logistic", w, partitions=world, threads=world)
    assert res["smooth"]["count"] == cnt == 6001
    assert abs(res["smooth"]["loss"] - loss) <= 1e-12 * abs(loss)
    np.testing.assert_allclose(res["smooth"]["grad"], g, rtol=0, atol=1e-12 * np.max(np.abs(g)))
    ref = O.agd_run(D, "logistic", "squared_l2", np.zeros(1024), convergence_tol=0.0, num_iterations=8, reg_param=0.01,
                    partitions=world, threads=world)
    r = res["run"]
    np.testing.assert_allclose(r["hist"], ref.loss_history, rtol=1e-11)
    assert np.linalg.norm(np.array(r["w"]) - ref.weights) <= 1e-9 * np.linalg.norm(ref.weights)
    assert (r["passes"], r["backtracks"], r["restarts"]) == (ref.passes, ref.backtracks, ref.restarts)
    assert r["collective_kind"] == 1 and r["collective_calls"] > 0       # the peer-memory exchange carried every pass
    # memoised (speculative two-gradient sweeps: twice the payload) and unfused runs: the same bits on every rank
    assert res["modes_bit_identical_on_every_rank"] is True and res["memo_fused_passes"] > 0
    # --- another dimension on the same handle (exchange rebuilt)
    X2, y2 = make_data(3000, 260, 9)
    l2, g2, c2 = O.smooth(O.Data(y2, X=X2.astype(np.float64)), "least_squares", np.full(260, 0.01), partitions=world, threads=world)
    assert res["smooth_d2"]["count"] == c2
    assert abs(res["smooth_d2"]["loss"] - l2) <= 1e-12 * abs(l2)
    np.testing.assert_allclose(res["smooth_d2"]["grad"], g2, rtol=0, atol=1e-12 * np.max(np.abs(g2)))
    # --- the synthetic workload generated in place: rank r holds rows [r*n/W, (r+1)*n/W) of the one global matrix
    Xs = O.synth_dense_f32(42, 0, 20000, 512)
    ys = O.synth_labels(42, "logistic", 0, Xs, O.synth_wtrue(42, 512))
    refs = O.agd_run(O.Data(ys, X=Xs), "logistic", "simple", np.zeros(512), convergence_tol=0.0, num_iterations=5,
                     partitions=world, threads=world)
    assert res["synthetic"]["rows_local"] == 20000 // world
    np.testing.assert_allclose(res["synthetic"]["hist"], refs.loss_history, rtol=1e-11)
    assert np.linalg.norm(np.array(res["synthetic"]["w"]) - refs.weights) <= 1e-9 * np.linalg.norm(refs.weights)
    assert res["synthetic"]["passes"] == refs.passes
    # --- mini-batch runs on bf16 shards (wgmma kernel): every rank but 0 samples with row_base != 0
    mb = res["minibatch_bf16_synthetic"]
    Xb = bf16_to_f32(f32_to_bf16_bits(Xs))
    rw, rh = O.gd_run(O.Data(np.array(mb["labels"]), X=Xb), "logistic", "squared_l2", np.zeros(512), step_size=0.5,
                      num_iterations=8, reg_param=0.01, partitions=world, threads=world, mini_batch_fraction=0.25)
    assert len(mb["hist"]) == len(rh) == 8
    np.testing.assert_allclose(mb["hist"], rh, rtol=1e-7)
    assert np.linalg.norm(np.array(mb["w"]) - rw) <= 1e-6 * np.linalg.norm(rw)
    # loaded shards number rank r's rows from r << 40: fp64 restatement of the same loop with that mask
    ml = res["minibatch_bf16_loaded"]
    Xl = bf16_to_f32(f32_to_bf16_bits(X)).astype(np.float64)
    ids = np.concatenate([(r << 40) + np.arange((r + 1) * 6001 // world - r * 6001 // world) for r in range(world)])
    wr, hr = np.zeros(1024), []
    for i in range(1, 7):
        sel = row_selected(42 + i, int(np.ldexp(0.25, 64)), ids)
        mult, lo = row_terms("logistic", Xl[sel] @ wr, y[sel])
        hr.append(lo.sum() / sel.sum())
        wr = wr - 0.5 / np.sqrt(i) * (Xl[sel].T @ mult / sel.sum())
    np.testing.assert_allclose(ml["hist"], hr, rtol=1e-7)
    assert np.linalg.norm(np.array(ml["w"]) - wr) <= 1e-6 * np.linalg.norm(wr)
    # the ring kernel on the generated shard, against the oracle (row ids = the oracle's)
    mr = res["minibatch_f32_ring_synthetic"]
    rw, rh = O.gd_run(O.Data(ys, X=Xs), "logistic", "squared_l2", np.zeros(512), step_size=0.5, num_iterations=8,
                      reg_param=0.01, partitions=world, threads=world, mini_batch_fraction=0.25)
    np.testing.assert_allclose(mr["hist"], rh, rtol=1e-10)
    assert np.linalg.norm(np.array(mr["w"]) - rw) <= 1e-9 * np.linalg.norm(rw)
    # every other kernel on loaded shards (rows from r << 40), with +-inf / NaN rows on ranks >= 1 that the mask always drops:
    # the fp64 restatement never reads those rows
    Xp, poisoned = minibatch_poisoned(X, world)
    assert len(poisoned) == 3 * (world - 1)
    thresh = int(np.ldexp(MB_FRACTION, 64))
    for key, kernel in (("f32_ring", "ring"), ("f64_generic", "generic"), ("bf16_ring", "ring"), ("csr_f32", "csr"),
                        ("csr_f64", "csr")):
        Xk = bf16_to_f32(f32_to_bf16_bits(Xp)).astype(np.float64) if key == "bf16_ring" else Xp.astype(np.float64)
        wr, hr = np.zeros(1024), []
        for i in range(1, MB_ITERS + 1):
            sel = row_selected(42 + i, thresh, ids)
            assert not sel[poisoned].any()
            mult, lo = row_terms("logistic", Xk[sel] @ wr, y[sel])
            hr.append(lo.sum() / sel.sum())
            wr = wr - 0.5 / np.sqrt(i) * (Xk[sel].T @ mult / sel.sum())
        mk = res["minibatch_loaded_" + key]
        assert kernel in mk["kernel"], (key, mk["kernel"])
        assert np.all(np.isfinite(mk["w"])), key
        np.testing.assert_allclose(mk["hist"], hr, rtol=1e-10, err_msg=key)
        assert np.linalg.norm(np.array(mk["w"]) - wr) <= 1e-9 * np.linalg.norm(wr), key
    # --- a wide sparse shard (d = 100000): the exchange takes its reduce-scatter + all-gather form (n >= 32768 doubles)
    rp, ix, va, y3 = make_csr(9000, 100000, 12, 13)
    D3 = O.Data(y3, csr=(rp, ix.ravel(), va.ravel()), d=100000)
    w3 = np.random.default_rng(17).standard_normal(100000) * 0.1
    l3, g3, c3 = O.smooth(D3, "hinge", w3, partitions=world, threads=world)
    wd = res["wide"]
    assert wd["count"] == c3 == 9000 and wd["collective_kind"] == 1
    assert abs(wd["loss"] - l3) <= 1e-12 * abs(l3)
    np.testing.assert_allclose(wd["grad"], g3, rtol=0, atol=1e-12 * np.max(np.abs(g3)))   # every element
    ref3 = O.agd_run(D3, "hinge", "squared_l2", np.zeros(100000), convergence_tol=0.0, num_iterations=5, reg_param=0.05,
                     partitions=world, threads=world)
    np.testing.assert_allclose(wd["hist"], ref3.loss_history, rtol=1e-10)
    np.testing.assert_allclose(wd["memo_hist"], ref3.loss_history, rtol=1e-10)
    assert abs(wd["w_l2"] - np.linalg.norm(ref3.weights)) <= 1e-9 * np.linalg.norm(ref3.weights)
    assert abs(wd["memo_w_l2"] - np.linalg.norm(ref3.weights)) <= 1e-9 * np.linalg.norm(ref3.weights)
    np.testing.assert_allclose(wd["w_head"], ref3.weights[:64], rtol=0, atol=1e-9 * np.max(np.abs(ref3.weights)))
