"""CPU-only checks of the Python side of the C ABI: the ctypes signature table and structs agree with
include/b200gsr.h, and inputs reach the kernels as they expect them (float32, contiguous, 16-byte aligned)."""
import contextlib
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from dreamscene_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200gsr.h")

_RETURNS = {"int": C.c_int, "size_t": C.c_size_t, "constchar*": C.c_char_p}
_SCALARS = {"int32_t": C.c_int32, "uint32_t": C.c_uint32, "uint64_t": C.c_uint64, "size_t": C.c_size_t,
            "float": C.c_float}
_STRUCTS = {"b200gsr_params": _lib.Params, "b200gsr_view_inputs": _lib.ViewInputs, "b200gsr_view_grads": _lib.ViewGrads,
            "b200gsr_group": _lib.Group, "b200gsr_group_grad": _lib.GroupGrad, "b200gsr_adam_tensor": _lib.AdamTensor,
            "b200gsr_saved_layout": _lib.SavedLayout, "b200gsr_scratch_layout": _lib.ScratchLayout}


def _prototypes():
    """{name: (return type, [argument declarations])} of every function the header declares."""
    src = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    src = re.sub(r"//[^\n]*", " ", src)
    out = {}
    for ret, name, args in re.findall(r"(const\s+char\s*\*|\bint|\bsize_t)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src):
        args = [" ".join(a.split()) for a in args.split(",")]
        out[name] = (ret.replace(" ", ""), [] if args == ["void"] else args)
    return out


def _is_pointer(t) -> bool:
    return t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer)


def _mismatches(signatures: dict, protos: dict) -> list:
    """Every disagreement between a signature table and the header: return type, argument count, and per argument
    its kind (pointer, pointer to the struct the binding mirrors, or the exact integer / float type)."""
    out = [("names", sorted(set(signatures) ^ set(protos)))] if set(signatures) != set(protos) else []
    for name in sorted(set(signatures) & set(protos)):
        (restype, argtypes), (ret, args) = signatures[name], protos[name]
        if restype is not _RETURNS[ret]:
            out.append((name, "return", ret))
        if len(argtypes) != len(args):
            out.append((name, "count", len(args)))
            continue
        for i, (t, decl) in enumerate(zip(argtypes, args)):
            if "*" in decl:
                pointee = decl.split("*")[0].replace("const ", "").strip()
                ok = _is_pointer(t) and (pointee not in _STRUCTS or t is C.POINTER(_STRUCTS[pointee]))
            else:
                ok = t is _SCALARS[decl.replace("const ", "").split()[0]]
            if not ok:
                out.append((name, i, decl))
    return out


def test_signature_table_matches_every_header_prototype():
    protos = _prototypes()
    assert len(protos) == 35 and list(_lib.SIGNATURES) == _lib.EXPORTS
    assert _mismatches(_lib.SIGNATURES, protos) == []


def test_signature_check_catches_any_single_wrong_entry():
    protos = _prototypes()
    # a 64-bit integer where a pointer belongs is the silent case: ctypes would pass it without complaint
    wrong = {C.c_int32: C.c_uint32, C.c_uint32: C.c_int32, C.c_uint64: C.c_uint32, C.c_float: C.c_int32}
    for name, (restype, argtypes) in _lib.SIGNATURES.items():
        for i, t in enumerate(argtypes):
            bad = argtypes[:i] + [C.c_uint64 if _is_pointer(t) else wrong[t]] + argtypes[i + 1:]
            assert _mismatches({**_lib.SIGNATURES, name: (restype, bad)}, protos) != [], (name, i)
        if argtypes:
            assert _mismatches({**_lib.SIGNATURES, name: (restype, argtypes[:-1])}, protos) != [], name
        assert _mismatches({**_lib.SIGNATURES, name: (C.c_uint32, argtypes)}, protos) != [], name
    pointers = dict(_lib.SIGNATURES)
    restype, argtypes = pointers["b200gsr_forward_views"]
    pointers["b200gsr_forward_views"] = (restype, [argtypes[0], argtypes[2], argtypes[1]] + argtypes[3:])
    assert _mismatches(pointers, protos) != []        # struct arrays swapped


def test_loaded_library_carries_the_signature_table():
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name


def test_struct_layouts_match_the_header_native_check(tmp_path):
    """tests/native/abi_layout_check.cu prints sizeof and every offsetof of the header's structs; the ctypes mirrors
    must agree field by field."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "abi_layout_check")
    src = os.path.join(ROOT, "tests", "native", "abi_layout_check.cu")
    subprocess.run([nvcc, "-std=c++17", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "include"), "-o", exe,
                    src], check=True, timeout=300)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stdout + out.stderr
    sizes, offsets = {}, {}
    for line in out.stdout.splitlines():
        struct, field, value = line.split()
        if field == "sizeof":
            sizes[struct] = int(value)
        else:
            offsets.setdefault(struct, {})[field] = int(value)
    assert set(sizes) == set(_STRUCTS)
    for struct, cls in _STRUCTS.items():
        assert C.sizeof(cls) == sizes[struct], struct
        assert {f: getattr(cls, f).offset for f, _ in cls._fields_} == offsets[struct], struct


def test_prepare_gives_float32_contiguous_16_byte_aligned_inputs():
    base = torch.arange(40, dtype=torch.float32)
    view = base[1:17].view(4, 4)                       # contiguous, 4 bytes past an aligned address
    assert view.is_contiguous() and view.data_ptr() % 16 == 4
    p = _lib.prepare(view)
    assert p.data_ptr() % 16 == 0 and p.is_contiguous() and p.dtype == torch.float32 and torch.equal(p, view)
    aligned = base[4:20].view(4, 4)
    assert _lib.prepare(aligned) is aligned            # nothing to do: no copy
    strided = base.double().view(4, 10)[:, 1:5]
    q = _lib.prepare(strided)
    assert q.dtype == torch.float32 and q.is_contiguous() and q.data_ptr() % 16 == 0 and torch.equal(q, strided.float())
    leaf = torch.randn(4, 4, dtype=torch.float64, requires_grad=True)
    assert _lib.prepare(leaf).grad_fn is not None      # not detached: autograd saves the prepared tensors
    assert _lib.prepare(None) is None


def test_densify_and_prune_passes_rotation_aligned_to_split_children(monkeypatch):
    """split_children reads the parents' rotations as float4: a rotation tensor at a misaligned storage offset must
    reach it through the preparation helper.  A fake library records what every entry point receives."""
    from dreamscene_b200 import densify
    P = 8
    calls = {}

    class FakeLib:
        def b200gsr_densify_scratch_bytes(self, n):
            return 64

        def __getattr__(self, name):
            def entry(*args):
                calls[name] = args
                if name == "b200gsr_densify_plan":               # keep every Gaussian, nothing cloned or split
                    (C.c_int32 * 5).from_address(args[11].value)[:] = [P, 0, 0, 0, P]
                if name == "b200gsr_split_children":             # the rotation rows, read while they are alive
                    calls["rotation_rows"] = list((C.c_float * (4 * P)).from_address(args[7].value))
                return 0
            return entry

    monkeypatch.setattr(_lib, "load", lambda: FakeLib())
    monkeypatch.setattr(_lib, "stream", lambda dev: None)
    monkeypatch.setattr(densify, "_cuda_device", lambda t: t.device)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    g = torch.Generator().manual_seed(0)
    rotation = torch.randn(4 * P + 1, generator=g)[1:].view(P, 4)
    assert rotation.data_ptr() % 16 == 4
    params = dict(xyz=torch.randn(P, 3, generator=g), f_dc=torch.randn(P, 1, 3, generator=g),
                  f_rest=torch.randn(P, 15, 3, generator=g), opacity=torch.randn(P, 1, generator=g),
                  scaling=torch.randn(P, 3, generator=g), rotation=rotation)
    densify.densify_and_prune(params, None, torch.zeros(P, 1), torch.ones(P, 1), 0.0002, 0.005, 1.0, None)
    rot_ptr = calls["b200gsr_split_children"][7].value
    assert rot_ptr % 16 == 0 and rot_ptr != rotation.data_ptr()
    assert calls["rotation_rows"] == rotation.reshape(-1).tolist()
