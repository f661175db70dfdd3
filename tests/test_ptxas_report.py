"""The conv kernel instantiations the YOLOv5-s, YOLOX-s, FCOS and DeepLab plans select compile without register spills and without
compiler-injected wgmma fences (tools/ptxas_report.py --check; compiles conv_tc.cu for sm_90a, no GPU needed)."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which('nvcc')), reason='needs nvcc')
def test_selected_conv_kernels_do_not_spill_or_fence():
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which('nvcc')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'ptxas_report.py'), '--check', '--nvcc', nvcc], capture_output=True,
                       text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
