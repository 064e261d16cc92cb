"""The group packer's routing rule and C ABI without a device (kr_shard_of_key, include/kr_engine.h; DESIGN §6).

A shard is FNV-1a 64 over namespace + "/" + RayCluster name, modulo the shard count: the same hash the native packer stores as
c_uid_hash for a RayCluster without a UID (tests/test_gpu_group_packer.py checks that equality on the device)."""
import os
import re

import pytest

from kuberay_b200 import abi
from kuberay_b200.packer import shard_of_key

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()


def fnv1a64(data: bytes) -> int:
    h = 0xCBF29CE484222325
    for b in data:
        h = ((h ^ b) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h


def py_shard(ns, name, n: int) -> int:
    enc = lambda v: b"" if v is None else (v if isinstance(v, bytes) else v.encode("utf-8"))  # noqa: E731
    return fnv1a64(enc(ns) + b"/" + enc(name)) % n


KEYS = [("default", "raycluster-0"), ("default", "raycluster-1"), ("team-a", "llm-serve"), ("kube-system", "x"), ("default", ""),
        ("", "rc"), ("", ""), ("default", None), ("ns-été", "clüster-漢字"), ("a" * 63, "b" * 253),
        (b"ns\xff\xfe", b"\x00name\x80"), ("default", "raycluster-with-a-long-name-0123456789abcdef")]


@pytest.mark.parametrize("n", range(1, 9))
def test_shard_of_key_is_fnv1a_of_ns_slash_name(n):
    for ns, name in KEYS:
        assert shard_of_key(ns, name, n) == py_shard(ns, name, n), (ns, name, n)
    for i in range(200):
        assert shard_of_key("default", f"raycluster-{i}", n) == py_shard("default", f"raycluster-{i}", n)


def test_shard_of_key_edges():
    assert fnv1a64(b"") == 0xCBF29CE484222325 and fnv1a64(b"a") == 0xAF63DC4C8601EC8C  # the published FNV-1a 64 test vectors
    assert shard_of_key("default", None, 5) == shard_of_key("default", "", 5)  # an absent label routes like ""
    assert shard_of_key("default", "rc", 0) == 0
    # the separator is part of the key: ("a", "b/c") and ("a/b", "c") hash alike (both are "a/b/c"); Kubernetes names have no "/"
    assert shard_of_key("a", "b/c", 7) == shard_of_key("a/b", "c", 7) == py_shard("a/b", "c", 7)
    # keys spread over the shards
    for n in (2, 3, 4, 8):
        hit = {shard_of_key("default", f"raycluster-{i}", n) for i in range(256)}
        assert hit == set(range(n)), n


def test_group_packer_section_of_the_header():
    declared = set(re.findall(r"^(?:const )?[a-z_0-9]+\s*\*?\s*(kr_(?:group_packer|shard_of_key)[a-z_0-9]*)\s*\(", HEADER, flags=re.M))
    assert declared == {"kr_shard_of_key", "kr_group_packer_create", "kr_group_packer_destroy", "kr_group_packer_size", "kr_group_packer_shard",
                        "kr_group_packer_group", "kr_group_packer_pod_upsert", "kr_group_packer_pod_delete", "kr_group_packer_cluster_upsert",
                        "kr_group_packer_cluster_delete", "kr_group_packer_job_upsert", "kr_group_packer_job_delete", "kr_group_packer_flush",
                        "kr_group_packer_reconcile", "kr_group_packer_last_error"}
    assert declared <= set(abi.ENGINE_SYMBOLS) | set(abi.ENGINE_HANDLE_SYMBOLS)
    assert re.search(r"kr_packer \*kr_group_packer_shard\(kr_group_packer \*gp, uint32_t shard\);", HEADER)
    assert re.search(r"kr_group\s+\*kr_group_packer_group\(kr_group_packer \*gp\);", HEADER)
    assert re.search(r"int\s+kr_group_packer_reconcile\(kr_group_packer \*gp, const kr_flags \*flags /\* \[n\] \*/, kr_results_view \*views /\* \[n\] \*/\);", HEADER)


def test_library_exports_the_handle_symbols(engine_lib):
    for name in abi.ENGINE_HANDLE_SYMBOLS:
        assert hasattr(engine_lib, name), name


def test_group_packer_create_rejects_bad_arguments(engine_lib):
    import ctypes as C
    cfg = abi.kr_config(0, 4, 4, 4, 4, 4, 4, 4, 4096)
    h = C.c_void_p()
    assert engine_lib.kr_group_packer_create(None, None, 1, C.byref(h)) == abi.KR_E_INVALID
    assert engine_lib.kr_group_packer_create(C.byref(cfg), None, 0, C.byref(h)) == abi.KR_E_INVALID
    assert engine_lib.kr_group_packer_create(C.byref(cfg), None, 65, C.byref(h)) == abi.KR_E_INVALID
    assert engine_lib.kr_group_packer_size(None) == 0 and engine_lib.kr_group_packer_shard(None, 0) is None
    assert engine_lib.kr_group_packer_last_error(None) == b"null group packer"
    assert engine_lib.kr_group_packer_flush(None, None) == abi.KR_E_INVALID
