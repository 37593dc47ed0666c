"""GPU: in every conv math mode, on the cfg2 ScanNet scene, the cfg5 SUNCG scene and ground-truth RoIs, every layer runs on
the same kernel route as recorded in tests/golden/conv_routes.json -- the ordered per-kernel timing names, the libsis3d
launch count of the forward and the conv3d_k3_tc_kernel instances of the mask stage (tools/capture_routes.py).  The capture
runs in a child process: profiling windows opened late in a long test process were seen to miss kernels."""
import json
import os
import subprocess
import sys

import pytest

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu


def test_every_layer_keeps_its_route(tmp_path):
    out = tmp_path / "routes.json"
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "capture_routes.py"), str(out)], capture_output=True,
                       text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-4000:]
    got = json.load(open(out))
    with open(os.path.join(GOLDEN, "conv_routes.json")) as f:
        want = json.load(f)
    assert set(got) == set(want)
    for case in want:
        assert got[case] == want[case], f"{case}: routes differ from the recorded ones"
