"""CPU: the host-side logic of ``engine/bbox_aug.im_detect_bbox_aug`` (pass order, flip / range / size of every collect, padding,
unpacking, the overflow error) over torch stand-ins of its three ops — in its own process, because the stand-ins monkey-patch
``mqdet_b200.ops`` and ``Tensor.is_cuda`` (tests/hostlogic/ops_double.py).  The kernels are checked by tests/test_bbox_aug_gpu.py."""
import os
import subprocess
import sys

from util import ROOT


def test_im_detect_bbox_aug_host_logic():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostlogic", "bbox_aug_case.py")], capture_output=True, text=True,
                       timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "PASS bbox_aug" in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])
