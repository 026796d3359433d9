"""Starts a process-per-rank world for the multi-rank GPU tests: one worker process per rank, as under torchrun / one Spark
executor per GPU.  Each worker is called as `worker.py rank world port device [extra ...] out`."""
import json
import os
import socket
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def run_world(worker, world, out, devices=None, extra=(), timeout=420):
    """Runs tests/<worker> as ranks 0 .. world - 1 (rank r on devices[r], device 0 by default) and returns the JSON the ranks
    wrote to `out`.  A rank that fails or hangs fails the test with the tail of every rank's log."""
    port = free_port()
    devices = devices or [0] * world
    env = dict(os.environ, OMP_NUM_THREADS="1")
    procs = [subprocess.Popen([sys.executable, os.path.join(HERE, worker), str(r), str(world), str(port), str(devices[r]),
                               *extra, out], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
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
