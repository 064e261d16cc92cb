"""The native event-driven packer (kr_packer_*, kuberay_b200/csrc/kr_packer.cpp; SURVEY §8(f) rank 1).

Object-level differential test: the same RayClusters / Pods / RayJobs (tests/fuzz_objects.py, drawn from the whole input domain)
go (a) through the Python packer into the CPU oracle and (b) event by event through the native packer into the engine it owns.
Ids and row numbers differ between the two (different interning order, free rows), so the records are compared through the
strings and Pod keys they stand for.  Then random informer events are applied to both; most epochs must be incremental
(pod rows / small tables only) and every epoch must still agree."""
import copy

import numpy as np
import pytest

from harness import PACKER_CAPS, Mirror, events, objects, packer_check, packer_stream
from kuberay_b200 import abi
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_native_packer_agrees_with_python_packer_and_stays_incremental(seed, oracle_mod):
    rng = np.random.default_rng(seed)
    clusters, pods, jobs = objects(seed, big=True)
    pk = Packer(**PACKER_CAPS)
    try:
        m = Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, pk)
        assert pk.flush() == abi.PACK_FULL
        packer_check(m, oracle_mod, lean=False)
        packer_check(m, oracle_mod, lean=True)
        e0, v0 = pk.epoch()
        counter = [0]
        _, modes = packer_stream(m, oracle_mod, 10, lambda epoch: events(rng, m, counter, structural=True), lean=lambda epoch: bool(epoch % 2))
        assert not any(mo & abi.PACK_FULL for mo in modes), modes
        e1, v1 = pk.epoch()
        assert e1 == e0 + 10 and v1 > v0
        assert any(mo & abi.PACK_POD_ROWS for mo in modes) and not all(mo & abi.PART_JSON for mo in modes)
        # a spec change bumps the generation: the JSON is re-emitted and travels; an unchanged generation does not re-emit
        key = sorted(m.clusters)[0]
        c = copy.deepcopy(m.clusters[key])
        c.pop("specJson", None)  # (from here on this RayCluster's hash input comes from the emitter, on both sides)
        c["spec"]["rayVersion"] = "9.9.9"; c["generation"] = 2; c["resourceVersion"] = 999
        m.upsert_cluster(c)
        assert pk.flush() & abi.PART_JSON
        packer_check(m, oracle_mod, lean=True)
        assert pk.cluster_epoch(pk.cluster_row(*key)) == (999, 2)
    finally:
        pk.close()
