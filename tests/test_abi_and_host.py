"""CPU tests: the C ABI surface (header <-> ctypes mirror <-> built library, no compute calls without a GPU), the oracle's
two List modes, the synthetic generator, UID-hash sharding, and the N>1 path over gloo (world_size 2)."""
import ctypes as C
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from kuberay_b200 import abi, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "kr_engine.h")


def test_library_exports_every_symbol_the_header_declares(engine_lib):
    text = open(HEADER).read()
    declared = set(re.findall(r"^(?:int|void|uint32_t|int64_t|kr_engine|const char) *\*? *(kr_[a-z_0-9]+)\s*\(", text, flags=re.M))
    assert declared == set(abi.ENGINE_SYMBOLS), declared ^ set(abi.ENGINE_SYMBOLS)
    for name in declared:
        assert hasattr(engine_lib, name), name


def test_struct_layouts_match_the_c_compiler():
    fields = {
        "kr_config": abi.kr_config, "kr_flags": abi.kr_flags, "kr_sizes": abi.kr_sizes, "kr_snapshot_bufs": abi.kr_snapshot_bufs,
        "kr_results_view": abi.kr_results_view, "kr_profile": abi.kr_profile,
    }
    records = {"kr_cluster_result": abi.cluster_result_dtype, "kr_group_result": abi.group_result_dtype, "kr_job_result": abi.job_result_dtype}
    prog = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', "int main(void){"]
    for n in list(fields) + list(records):
        prog.append(f'printf("{n} %zu\\n", sizeof({n}));')
    for f, _ in abi.cluster_result_dtype.fields.items():
        prog.append(f'printf("kr_cluster_result.{f} %zu\\n", offsetof(kr_cluster_result, {f}));')
    for f, _ in abi.group_result_dtype.fields.items():
        prog.append(f'printf("kr_group_result.{f} %zu\\n", offsetof(kr_group_result, {f}));')
    prog.append("return 0;}")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "t.c"), os.path.join(d, "t")
        open(src, "w").write("\n".join(prog))
        subprocess.check_call(["gcc", "-o", exe, src])
        out = dict(line.split() for line in subprocess.check_output([exe], text=True).splitlines())
    for n, t in fields.items():
        assert int(out[n]) == C.sizeof(t), n
    for n, dt in records.items():
        assert int(out[n]) == dt.itemsize, n
    for f, (_, off) in abi.cluster_result_dtype.fields.items():
        assert int(out[f"kr_cluster_result.{f}"]) == off, f
    for f, (_, off) in abi.group_result_dtype.fields.items():
        assert int(out[f"kr_group_result.{f}"]) == off, f


def test_enum_values_match_the_header():
    text = open(HEADER).read()
    vals = dict(re.findall(r"\b(KR_[A-Z0-9_]+)\s*=\s*(1u << \d+|-?\d+)\b", text))
    for cname, v in vals.items():
        pyname = cname[3:]
        if not hasattr(abi, pyname):
            continue
        want = (1 << int(v.split("<<")[1])) if "<<" in v else int(v)
        assert getattr(abi, pyname) == want, cname


def test_engine_refuses_to_run_without_a_gpu(engine_lib):
    """No CPU fallback: on a box without a device the product path raises instead of silently computing on the host."""
    from kuberay_b200.engine import Engine, EngineError
    if engine_lib.kr_device_count() > 0:
        pytest.skip("a CUDA device is visible here")
    with pytest.raises(EngineError):
        Engine(0, max_clusters=1)


def test_oracle_list_modes_and_threads_agree(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C2", groups=2, jobs=True))
    a = oracle_mod.run(snap, flags, list_mode=oracle_mod.INDEXED, threads=1)
    b = oracle_mod.run(snap, flags, list_mode=oracle_mod.NS_SCAN, threads=3)
    c = oracle_mod.run(snap, flags, list_mode=oracle_mod.INDEXED, threads=8)
    assert not a.diff(b) and not a.diff(c)
    assert a.n_actions > 0 and a.n_create_total > 0 and a.n_orphans > 0
    assert set(np.unique(a.clusters["path"])) >= {abi.PATH_NORMAL, abi.PATH_SKIPPED}


def test_synthetic_generator_is_deterministic_and_valid():
    s1, _ = synthetic.generate(synthetic.config("C1"))
    s2, _ = synthetic.generate(synthetic.config("C1"))
    for name, *_ in abi.COLUMNS:
        assert np.array_equal(s1.cols[name], s2.cols[name]), name
    assert s1.dims["clusters"] == 10 and s1.dims["pods"] == 40
    s1.validate()


def test_empty_and_ragged_snapshots(oracle_mod):
    from kuberay_b200.snapshot import pack_objects
    snap, meta = pack_objects([], [])
    res = oracle_mod.run(snap, meta.flags)
    assert res.n_actions == 0 and res.n_orphans == 0
    # a cluster with no pods at all, and pods with no cluster
    cl = {"namespace": "default", "name": "lonely", "spec": {"headGroupSpec": {"rayStartParams": {}}, "workerGroupSpecs": []}, "specJson": "{}"}
    pods = [{"namespace": "default", "name": "stray", "labels": {"ray.io/cluster": "gone", "ray.io/node-type": "worker"}, "phase": "Running"},
            {"namespace": "default", "name": "unlabelled", "labels": {}, "phase": "Running"}]
    snap, meta = pack_objects([cl], pods)
    res = oracle_mod.run(snap, meta.flags)
    assert res.n_orphans == 2 and res.clusters[0]["head_action"] == abi.HEAD_CREATE and res.clusters[0]["n_pods"] == 0
    assert list(res.sorted_action) == [abi.ACT_ORPHAN, abi.ACT_ORPHAN]


def test_uid_hash_sharding_reproduces_the_global_decisions(oracle_mod):
    """SURVEY §8(e): decisions need no exchange — every shard's records equal the global pass restricted to its clusters."""
    snap, flags = synthetic.generate(synthetic.config("C2", groups=2))
    glob = oracle_mod.run(snap, flags)
    world = 4
    seen = 0
    for rank in range(world):
        sh = synthetic.shard_by_uid(snap, rank, world)
        res = oracle_mod.run(sh, flags)
        keep = (snap.c_uid_hash % np.uint64(world)) == np.uint64(rank)
        want = glob.clusters[keep]
        for fld in ("path", "head_action", "err_kind", "err_arg", "stop_after_group", "n_pods", "n_heads", "new_state", "needs_status_write", "counts", "cond_status"):
            assert np.array_equal(res.clusters[fld], want[fld]), (rank, fld)
        assert np.array_equal(res.hash, glob.hash[keep])
        gkeep = keep[snap.g_cluster_idx]
        for fld in ("expected", "n_list", "n_unhealthy", "n_running", "diff", "n_create", "flags"):
            assert np.array_equal(res.groups[fld], glob.groups[gkeep][fld]), (rank, fld)
        seen += sh.dims["clusters"]
    assert seen == snap.dims["clusters"]


GLOO_WORKER = r'''
import os, sys
sys.path.insert(0, sys.argv[1])
import numpy as np, torch, torch.distributed as dist
from kuberay_b200 import abi, synthetic
from oracle import oracle
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=400))
shard = synthetic.shard_by_uid(snap, rank, world)
res = oracle.run(shard, flags)
# the optional exchange step: all-gather the per-group delta records (32 B each), padded to the largest shard
ng = torch.tensor([shard.dims["groups"]]); dist.all_reduce(ng, op=dist.ReduceOp.MAX)
buf = torch.zeros(int(ng) * 32, dtype=torch.uint8)
raw = torch.from_numpy(res.groups.view(np.uint8).copy())
buf[:raw.numel()] = raw
out = [torch.zeros_like(buf) for _ in range(world)]
dist.all_gather(out, buf)
counts = [torch.zeros(1, dtype=torch.int64) for _ in range(world)]
dist.all_gather(counts, torch.tensor([shard.dims["groups"]]))
if rank == 0:
    glob = oracle.run(snap, flags)
    total_diff = 0
    for r in range(world):
        n = int(counts[r])
        g = out[r][: n * 32].numpy().view(abi.group_result_dtype)
        keep = ((snap.c_uid_hash % np.uint64(world)) == np.uint64(r))[snap.g_cluster_idx]
        assert np.array_equal(g["diff"], glob.groups[keep]["diff"]) and np.array_equal(g["n_create"], glob.groups[keep]["n_create"])
        total_diff += int(g["diff"].sum())
    assert total_diff == int(glob.groups["diff"].sum())
    print("GLOO_OK", total_diff)
dist.destroy_process_group()
'''


def test_two_rank_gloo_sharded_pass_and_delta_allgather():
    """The N>1 path on CPU: torch.distributed (gloo), world_size 2, UID-hash shards, all-gather of the group delta records."""
    with tempfile.TemporaryDirectory() as d:
        script = os.path.join(d, "w.py")
        open(script, "w").write(GLOO_WORKER)
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", "29517", script, ROOT]
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert "GLOO_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]


def test_results_diff_reports_create_runs_that_overlap_or_leave_the_list():
    """Results.diff compares the replica-index arena group by group through (create_off, n_create).  Runs that share places or
    run past the end of create_idx are a fault of the producer, even where the values they read happen to agree."""
    sizes = abi.kr_sizes(n_clusters=1, n_groups=3, n_wtd=0, n_pods=0, n_heads=0, n_jobs=0, json_bytes=0)

    def results(offs, cnts, idx):
        r = abi.Results(sizes, len(idx))
        r.groups["create_off"], r.groups["n_create"] = offs, cnts
        r.create_idx[:] = idx
        r.n_create_total = int(sum(cnts))
        return r

    want = results([0, 2, 4], [2, 2, 1], [0, 1, 0, 1, 7])
    assert not want.diff(results([3, 1, 0], [2, 2, 1], [7, 0, 1, 0, 1]))   # another layout of the same runs
    # groups 0 and 1 share their two places: the values agree ([0, 1] both), only the layout check sees it
    overlap = results([0, 0, 4], [2, 2, 1], [0, 1, 9, 9, 7])
    d = want.diff(overlap)
    assert any("overlap or leave the list" in m for m in d), d
    # a run past the end of the list
    past = results([0, 2, 4], [2, 2, 1], [0, 1, 0, 1, 7])
    past.groups["create_off"][2] = 5
    d = want.diff(past)
    assert any("overlap or leave the list" in m for m in d), d
    assert any("overlap or leave the list" in m for m in past.diff(want))
    # an empty group may sit anywhere, even at the end of the list
    empty = results([0, 2, 4], [2, 2, 1], [0, 1, 0, 1, 7])
    empty.groups["n_create"][2], empty.n_create_total = 0, 4
    want_empty = results([0, 2, 99], [2, 2, 0], [0, 1, 0, 1, 7])
    want_empty.n_create_total = 4
    assert not want_empty.diff(empty)
