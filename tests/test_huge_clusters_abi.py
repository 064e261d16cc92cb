"""The huge-RayCluster option without a device: its constant in the Python bindings matches include/kr_engine.h, the Go shim
declares it, and the C3H workload has the shape its benchmark expects."""
import os
import re

from kuberay_b200 import abi, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()


def test_option_constant_matches_the_header():
    assert int(re.search(r"KR_OPT_HUGE_CLUSTERS\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_HUGE_CLUSTERS == 6


def test_go_shim_declares_the_option():
    src = open(os.path.join(ROOT, "integration", "go", "krengine", "engine.go")).read()
    assert re.search(r"OptHugeClusters\s*=\s*uint32\(C\.KR_OPT_HUGE_CLUSTERS\)", src)


def test_c3h_shape():
    p = synthetic.config("C3H")
    assert (p.n_clusters, p.pods_per_cluster, p.n_large, p.large_pods) == (10000, 100, 2, 20000)
    assert p.large_pods > abi.LARGE_MAX_PODS
