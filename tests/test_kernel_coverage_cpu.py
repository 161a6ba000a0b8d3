"""Every C entry point of include/ctrlora_b200.h is exercised by at least one GPU test.

An entry point counts as tested when a `tests/test_*_gpu.py` file calls it by its C name (`lib.ctrlora_x(...)`) or
calls an `ops.<wrapper>(...)` whose body -- directly or through other wrappers of ctrlora_b200/ops.py -- names it.
The GPU tests themselves need a device; this check reads source only, so it runs everywhere and fails with the names of
the entry points that no GPU test reaches, e.g. a new export added without a test.
"""
import ast
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")

# entry point -> why no GPU test has to call it
ALLOWED = {
    "ctrlora_abi_version": "no device work: checked by tests/test_host_cpu.py and by the build",
}


def header_entry_points():
    with open(os.path.join(ROOT, "include", "ctrlora_b200.h")) as f:
        src = f.read()
    return set(re.findall(r"^\s*int\s+(ctrlora_\w+)\s*\(", src, flags=re.M))


def wrapper_entry_points():
    """ops.<function> -> the entry points it reaches (attributes named ctrlora_*, followed through calls of other ops
    functions)."""
    with open(os.path.join(ROOT, "ctrlora_b200", "ops.py")) as f:
        tree = ast.parse(f.read())
    funcs = {n.name: n for n in tree.body if isinstance(n, ast.FunctionDef)}
    direct, calls = {}, {}
    for name, fn in funcs.items():
        direct[name] = {n.attr for n in ast.walk(fn) if isinstance(n, ast.Attribute) and n.attr.startswith("ctrlora_")}
        calls[name] = {n.func.id for n in ast.walk(fn)
                       if isinstance(n, ast.Call) and isinstance(n.func, ast.Name) and n.func.id in funcs}
    reach = {}
    for name in funcs:
        seen, todo, eps = set(), [name], set()
        while todo:
            f = todo.pop()
            if f in seen:
                continue
            seen.add(f)
            eps |= direct[f]
            todo.extend(calls[f])
        reach[name] = eps
    return reach


def gpu_test_calls(path):
    """(C names called, ops wrappers called) in one test file"""
    with open(path) as f:
        tree = ast.parse(f.read())
    c_names, wrappers = set(), set()
    for n in ast.walk(tree):
        if isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute):
            if n.func.attr.startswith("ctrlora_"):
                c_names.add(n.func.attr)
            elif isinstance(n.func.value, ast.Name) and n.func.value.id == "ops":
                wrappers.add(n.func.attr)
    return c_names, wrappers


def reached_entry_points(skip=()):
    reach = wrapper_entry_points()
    got = set()
    for fname in sorted(os.listdir(TESTS)):
        if not (fname.startswith("test_") and fname.endswith("_gpu.py")) or fname in skip:
            continue
        c_names, wrappers = gpu_test_calls(os.path.join(TESTS, fname))
        got |= c_names
        for w in wrappers:
            got |= reach.get(w, set())
    return got


def test_header_parse_finds_the_exports():
    eps = header_entry_points()
    from ctrlora_b200 import _lib
    int_exports = set(_lib.EXPORTS) - {"ctrlora_last_cuda_error"}  # the one export that returns a string
    assert eps == int_exports, (sorted(eps - int_exports), sorted(int_exports - eps))
    assert set(ALLOWED) <= eps, sorted(set(ALLOWED) - eps)


def test_wrapper_map():
    reach = wrapper_entry_points()
    assert reach["gemm"] == {"ctrlora_gemm_f16", "ctrlora_gemm_f16_simt"}
    assert reach["zeros"] == {"ctrlora_memset_zero"}
    assert reach["timestep_embedding"] == {"ctrlora_timestep_embedding", "ctrlora_timestep_embedding_f32"}
    assert reach["dpm_multistep_update"] == {"ctrlora_dpm_multistep_update"}


def test_every_entry_point_has_a_gpu_test():
    missing = sorted(header_entry_points() - set(ALLOWED) - reached_entry_points())
    assert not missing, f"entry points no tests/test_*_gpu.py reaches: {', '.join(missing)}"


def test_the_check_notices_a_missing_test():
    """Without the conditioning-kernel tests, the entry points only they reach are reported."""
    missing = header_entry_points() - set(ALLOWED) - reached_entry_points(skip=("test_conditioning_kernels_gpu.py",))
    assert {"ctrlora_cast_rows_f32_to_f16", "ctrlora_clip_embed", "ctrlora_dpm_multistep_update", "ctrlora_im2col_s2_f16",
            "ctrlora_quick_gelu_f16"} <= missing, sorted(missing)
