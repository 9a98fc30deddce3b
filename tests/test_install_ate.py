"""install() rebinds the reference's compute_ate (flowmap.misc.ate) when that module is present."""
import subprocess
import sys

from conftest import ROOT
from test_abi import _REFERENCE_STANDIN


def test_install_rebinds_compute_ate():
    code = _REFERENCE_STANDIN + (
        "module('flowmap.misc')\n"
        "ref_ate = module('flowmap.misc.ate', compute_ate=placeholder)\n"
        "import flowmap_b200\n"
        "rep = flowmap_b200.install()\n"
        "from flowmap_b200 import ate\n"
        "assert ref_ate.compute_ate is ate.compute_ate\n"
        "assert rep['flowmap.misc.ate.compute_ate'] is placeholder\n"
        "assert 'flowmap.visualization.visualizer_trajectory.compute_ate' not in rep\n")
    subprocess.check_call([sys.executable, "-c", code], cwd=str(ROOT))
