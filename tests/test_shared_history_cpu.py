"""CPU: b200dd_pipeline_share_history's binding matches the header, and the argument checks that need no pipeline
refuse before any CUDA call."""
import ctypes as C
import os
import re

from blah2_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_binding_matches_the_header():
    text = open(os.path.join(ROOT, "include", "b200dd.h")).read()
    decl = re.search(r"B200DD_API\s+(\w+)\s+b200dd_pipeline_share_history\s*\(([^)]*)\)", text)
    assert decl is not None
    assert decl.group(1) == "int"
    params = [p.strip() for p in decl.group(2).split(",")]
    assert params == ["b200dd_pipeline *const *members", "uint32_t n"]
    sig = {name: (res, args) for name, res, args in capi.SIGNATURES}["b200dd_pipeline_share_history"]
    assert sig[0] is C.c_int
    assert sig[1] == [C.c_void_p, C.c_uint32]


def test_bad_arguments_fail_before_any_cuda_call():
    lib = capi.load()
    assert lib.b200dd_pipeline_share_history(None, 0) == capi.ERR_ARG
    assert lib.b200dd_pipeline_share_history(None, 3) == capi.ERR_ARG
    members = (C.c_void_p * 2)(None, None)
    assert lib.b200dd_pipeline_share_history(members, 0) == capi.ERR_ARG
    assert lib.b200dd_pipeline_share_history(members, 2) == capi.ERR_ARG
    assert "null member" in capi.last_error()
