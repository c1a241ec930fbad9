"""The ctypes declarations in `gllm_b200.ops.lib` agree with the CUDA sources the library is built from.

ctypes checks Python callers against the declared parameter types, never those types against the C prototype;
a drifted declaration passes a wrong stride, pointer or stream on the GPU. This parses every source that
`gllm_b200.build` compiles and checks the exported entry points, their parameter types, the struct mirrors and
the mirrored limits. It cannot see two swapped parameters (or fields) of the same type; the GPU element-wise tests
cover what each argument means. Needs no nvcc, no library and no GPU.
"""
import ctypes
import re

import pytest

from gllm_b200 import build
from gllm_b200.ops import lib, sm100
from gllm_b200.parallel import fused

SCALARS = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "uint32_t": ctypes.c_uint32,
           "uint64_t": ctypes.c_uint64, "float": ctypes.c_float}
STRUCTS = {s.__name__: s for s in (lib.GemmComm, lib.ReduceNormArgs, lib.LLArgs, lib.NvlsArgs, lib.EpArgs)}


def _strip_comments(src):
    return re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", src, flags=re.S))


SRC = "\n".join(_strip_comments(open(p).read()) for p in build._sources())
PROTOS = {m[1]: [" ".join(p.split()) for p in m[2].split(",") if p.strip()]
          for m in re.finditer(r"GLLM_EXPORT\s+int\s+(gllm_\w+)\s*\(([^)]*)\)", SRC)}
BODIES = {m[1]: m[2] for m in re.finditer(r"\bstruct\s+(\w+)\s*\{([^}]*)\};", SRC) if m[1] in STRUCTS}


def _const(name):
    vals = set(re.findall(rf"constexpr\s+int\s+{name}\s*=\s*(\d+)\s*;", SRC))
    assert len(vals) == 1, f"{name}: expected one definition in csrc, found values {sorted(vals)}"
    return int(vals.pop())


def _ctype(what, base, ptr, in_struct=False):
    """C type `[const] base[*]` -> the ctypes type lib must declare for it."""
    if ptr:
        return ctypes.c_void_p if in_struct or base not in STRUCTS else ctypes.POINTER(STRUCTS[base])
    assert base in SCALARS, f"{what}: C type `{base}` has no ctypes mapping"
    return SCALARS[base]


def test_exported_entry_points_match_the_table():
    assert len(PROTOS) > 40, "the prototype parser found too few GLLM_EXPORT entry points"
    assert set(PROTOS) == set(lib.ABI), (f"exported but not declared in lib.ABI: {sorted(set(PROTOS) - set(lib.ABI))}; "
                                         f"declared but not exported: {sorted(set(lib.ABI) - set(PROTOS))}")


@pytest.mark.parametrize("name", sorted(PROTOS))
def test_parameter_types_match_the_prototype(name):
    declared = lib.ABI.get(name)
    assert declared is not None, f"{name} is not declared in lib.ABI"
    params = PROTOS[name]
    assert len(declared) == len(params), f"{name}: C takes {len(params)} parameters {params}, lib.ABI {len(declared)}"
    for i, (param, got) in enumerate(zip(params, declared)):
        m = re.fullmatch(r"(?:const )?(\w+) ?(\*?) ?\w+", param)
        assert m, f"{name}: cannot parse parameter {i} `{param}`"
        want = _ctype(f"{name} parameter {i} `{param}`", m[1], m[2])
        assert got is want, f"{name}: parameter {i} `{param}` is {want.__name__}, lib.ABI declares {got.__name__}"


@pytest.mark.parametrize("struct", sorted(STRUCTS))
def test_struct_mirror_matches_the_c_layout(struct):
    assert struct in BODIES, f"struct {struct} not found in csrc"
    want = []
    for decl in filter(None, (" ".join(d.split()) for d in BODIES[struct].split(";"))):
        m = re.fullmatch(r"(?:const )?(\w+) ?(\*?) ?(.+)", decl)
        assert m, f"{struct}: cannot parse `{decl}`"
        for d in m[3].split(","):
            f = re.fullmatch(r"(\w+)(?:\[(\w+)\])?", d.strip())
            assert f, f"{struct}: cannot parse declarator `{d}` of `{decl}`"
            n = None if f[2] is None else int(f[2]) if f[2].isdigit() else _const(f[2])
            want.append(_field(f[1], _ctype(f"{struct}.{f[1]}", m[1], m[2], in_struct=True), n))
    got = [_field(name, t._type_, t._length_) if issubclass(t, ctypes.Array) else _field(name, t, None)
           for name, t in STRUCTS[struct]._fields_]
    for i in range(max(len(want), len(got))):
        w, g = want[i] if i < len(want) else "nothing", got[i] if i < len(got) else "nothing"
        assert w == g, f"{struct} field {i}: C has {w}, the ctypes mirror has {g}"


def _field(name, t, n):
    return f"`{name}` {t.__name__}" + ("" if n is None else f"[{n}]")


def test_mirrored_limits_match_the_c_constants():
    assert lib.MAX_PEERS == _const("kMaxPeers") == _const("kMaxTp") == _const("kMaxEp")
    assert fused.MAX_BLOCKS == _const("kMaxBlocks")
    assert sm100.MAX_LOGPROBS == _const("kMaxLogprobs")
