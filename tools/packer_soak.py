#!/usr/bin/env python
"""A longer run of the native packer's random informer-event streams than tests/test_packer.py affords (4 seeds x 10 epochs there): per seed a
fuzz-generated object set, then epochs of mixed Pod / RayCluster / RayJob events — structural ones included — through kr_packer_*, every
epoch compared with the oracle on an independently re-packed snapshot (tests/harness.py's Mirror / packer_check).  usage (GPU box):
python tools/packer_soak.py [first_seed] [seeds] [epochs] [--all-options] [--bucket-pod-lists] [--json-bytes N] [--lean]

At the end it prints how many passes were incremental and full, and how often each KR_FULL_* cause sent a pass to the full pass
(kr_last_pass) — counts over synthetic streams, the input for choosing the options' defaults.
--all-options turns on all nine opt-in engine options (large / wide / huge RayClusters, workersToDelete edits, spec rows, RayCluster
creates and deletes, group edits, large growth) and adds spec edits with a bumped generation to every epoch
(tests/test_gpu_packer_streams.py and tests/test_gpu_structural_streams.py run these options at suite length); --json-bytes sets
kr_config.max_json_bytes, small enough (a few KiB above the fleet's muted specs) that the stream compacts the JSON arena as it goes;
--lean keeps fetch_pod_lists at 0 (by default every third epoch fetches the full pod lists, which takes the full pass twice), so the
histogram counts only what the events and options cause; --bucket-pod-lists turns on KR_OPT_BUCKET_POD_LISTS instead, with which the
fetching epochs keep the bucket pipeline and their incremental epochs."""
import argparse
import collections
import copy
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from harness import PACKER_CAPS, Mirror, events, objects, packer_check, spec_edits  # noqa: E402
from kuberay_b200 import abi  # noqa: E402
from kuberay_b200.packer import Packer  # noqa: E402
from oracle import oracle  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("first", nargs="?", type=int, default=10)
ap.add_argument("seeds", nargs="?", type=int, default=40)
ap.add_argument("epochs", nargs="?", type=int, default=30)
ap.add_argument("--all-options", action="store_true")
ap.add_argument("--json-bytes", type=int, default=4 << 20)
ap.add_argument("--lean", action="store_true")
ap.add_argument("--bucket-pod-lists", action="store_true")
a = ap.parse_args()
opts = dict(large_clusters=True, wide_clusters=True, huge_clusters=True, wtd_edits=True, spec_rows=True, cluster_creates=True,
            cluster_deletes=True, group_edits=True, large_growth=True) if a.all_options else {}
if a.bucket_pod_lists:
    opts["bucket_pod_lists"] = True
oracle.lib()
total = inc = 0
kinds, causes = collections.Counter(), collections.Counter()


def tally(pk):
    rep = pk.last_pass()
    kinds[rep["kind"]] += 1
    causes.update(rep["why"])


for seed in range(a.first, a.first + a.seeds):
    rng = np.random.default_rng(seed)
    clusters, pods, jobs = objects(seed, big=True)
    pk = Packer(**dict(PACKER_CAPS, max_pods=8192, max_json_bytes=a.json_bytes), **opts)
    try:
        m = Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, pk)
        assert pk.flush() == abi.PACK_FULL
        packer_check(m, oracle, lean=True)
        tally(pk)
        counter, gen = [0], [2]
        for epoch in range(a.epochs):
            if a.all_options:
                spec_edits(rng, m, gen, int(rng.integers(1, 4)))
            events(rng, m, counter, structural=True)
            mode = pk.flush()
            assert not mode & abi.PACK_FULL, (seed, epoch)
            packer_check(m, oracle, lean=a.lean or bool(epoch % 3))
            tally(pk)
            total += 1
            inc += bool(mode & abi.PACK_POD_ROWS)
    finally:
        pk.close()
print(f"packer soak ok: seeds {a.first}..{a.first + a.seeds - 1} x {a.epochs} epochs = {total} epochs ({inc} with pod-row commits), "
      f"options {'all on' if a.all_options else 'default'}, max_json_bytes {a.json_bytes}, every one equal to the oracle")
print(f"passes: {dict(kinds)}; full-pass causes (KR_FULL_*, a pass may have several): {dict(causes.most_common())}")
