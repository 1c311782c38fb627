"""CPU: the host-side logic of ``engine/lvis_eval.LvisEvaluatorFixedAP`` (slots, arrivals, sizes, cuts, label table, errors,
summary) over stand-ins of its three ops — in its own process, because the stand-ins monkey-patch ``mqdet_b200.ops`` and
``Tensor.is_cuda`` (tests/hostlogic/ops_double.py).  The kernels are checked by tests/test_lvis_eval_gpu.py."""
import os
import subprocess
import sys

from util import ROOT


def test_lvis_evaluator_host_logic():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostlogic", "lvis_eval_case.py")], capture_output=True, text=True,
                       timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "PASS lvis_eval" in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])
