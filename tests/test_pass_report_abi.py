"""CPU tests of kr_last_pass's surface: kr_pass_report and the KR_PASSK_* / KR_PIPE_* / KR_FULL_* constants in include/kr_engine.h,
their ctypes mirror in kuberay_b200/abi.py, the Go shim's use of them, and the names Engine.last_pass decodes why_full into."""
import ctypes as C
import os
import re

from kuberay_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()
GO = {f: open(os.path.join(ROOT, "integration", "go", "krengine", f)).read() for f in ("engine.go", "batcher.go")}


def header_enum(prefix: str) -> dict[str, int]:
    """KR_<prefix>* enumerators of the header, by name (their values are plain integers or 1u << n)."""
    out = {}
    for name, val in re.findall(r"\b(KR_" + prefix + r"[A-Z_0-9]*)\s*=\s*(1u\s*<<\s*\d+|\d+)", HEADER):
        m = re.fullmatch(r"1u\s*<<\s*(\d+)", val.strip())
        out[name] = 1 << int(m.group(1)) if m else int(val.strip().rstrip("u"))
    return out


def test_struct_layout_matches_the_header():
    m = re.search(r"typedef struct kr_pass_report\s*\{(.*?)\}\s*kr_pass_report;", HEADER, re.S)
    assert m
    body = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S)
    decls = [tuple(d.split()) for d in body.split(";") if d.strip()]
    assert [name for _t, name in decls] == [f for f, _ in abi.kr_pass_report._fields_]
    sizes = {"uint8_t": 1, "uint32_t": 4}
    off = 0
    for (typ, name), (field, ctype) in zip(decls, abi.kr_pass_report._fields_):
        off = (off + sizes[typ] - 1) // sizes[typ] * sizes[typ]
        assert getattr(abi.kr_pass_report, field).offset == off, field
        assert C.sizeof(ctype) == sizes[typ], field
        off += sizes[typ]
    assert C.sizeof(abi.kr_pass_report) == off == 16
    assert re.search(r"^int kr_last_pass\(kr_engine \*e, kr_pass_report \*out\);", HEADER, re.M)
    assert "kr_last_pass" in abi.ENGINE_SYMBOLS


def test_constants_match_the_header():
    assert header_enum("PASSK_") == {"KR_PASSK_INCREMENTAL": abi.PASSK_INCREMENTAL, "KR_PASSK_FULL": abi.PASSK_FULL}
    assert header_enum("PIPE_") == {"KR_PIPE_BUCKET": abi.PIPE_BUCKET, "KR_PIPE_SORT": abi.PIPE_SORT, "KR_PIPE_RADIX": abi.PIPE_RADIX}
    full = header_enum("FULL_")
    assert full == {"KR_FULL_" + k: v for k, v in abi.FULL_BITS.items()}
    assert list(full.values()) == [1 << i for i in range(len(full))]  # distinct bits, in declaration order
    for k, v in abi.FULL_BITS.items():
        assert getattr(abi, "FULL_" + k) == v


def test_full_names_decode_every_bit():
    assert abi.full_names(0) == []
    assert abi.full_names(abi.FULL_FIRST | abi.FULL_ARENA) == ["FIRST", "ARENA"]
    assert abi.full_names(sum(abi.FULL_BITS.values())) == list(abi.FULL_BITS)
    assert abi.full_names(1 << 31) == ["BIT31"]


def test_go_shim_reads_the_report_and_names_every_cause():
    eng, bat = GO["engine.go"], GO["batcher.go"]
    assert re.search(r"C\.kr_last_pass\(e\.h, &r\)", eng)
    assert "r.kind == C.KR_PASSK_INCREMENTAL" in eng
    named = set(re.findall(r"\{C\.(KR_FULL_[A-Z_]+),", eng))
    assert named == {"KR_FULL_" + k for k in abi.FULL_BITS}, named ^ {"KR_FULL_" + k for k in abi.FULL_BITS}
    # the batcher counts every epoch's pass: incremental / full, and each cause of a full one
    assert "b.p.Engine().LastPass()" in bat and "func (b *Batcher) Stats() Stats" in bat
    assert re.search(r"for _, c := range FullCauses", bat)
