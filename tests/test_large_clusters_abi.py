"""The large-RayCluster option's constants in the Python bindings match include/kr_engine.h (no device needed)."""
import os
import re

from kuberay_b200 import abi

HEADER = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "kr_engine.h")).read()


def test_option_constants_match_the_header():
    assert int(re.search(r"KR_OPT_LARGE_CLUSTERS\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_LARGE_CLUSTERS
    assert int(re.search(r"KR_OPT_BUCKET_STRIDE\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_BUCKET_STRIDE
    assert int(re.search(r"KR_LARGE_MAX_PODS\s*=\s*(\d+)", HEADER).group(1)) == abi.LARGE_MAX_PODS
