"""The configuration switches of the exact SIMT kernels, restated from the sources, and the shape lists of
test_exact_route_gpu.py that must straddle each of them (no GPU needed).

Each switch is read from the CUDA source where it is defined (a constant, or the arithmetic of a launcher), so that a
change of the kernels that moves a switch fails here until the GPU sweep follows it:

| switch | kernel | boundary |
|---|---|---|
| `exact_cfg`: 128 / 64 / 32-row tiles, then no staging | `exact_pass_kernel` | D = 381 / 382, 771 / 772, 1536 / 1537 |
| `kFewRows` | `exact_rows_few_kernel` / list mode of `exact_pass_kernel` | lists of 8192 / 8193 rows |
| `kKnnMaxSmemD` | `knn_warp_search_kernel` | D = 2048 / 2049 |
| 48 KB without opting in, minus 4 KB of static shared memory | `exact_rows_few_kernel`, `yy_rows_cta_kernel` | D = 11264 / 11265 |
| `kRowStageMaxD` | `exact_rows_few_kernel`, `yy_rows_cta_kernel` | D = 16384 / 16385 |
| `kStrictMaxD` | `strict_adjust_kernel` | D = 1600 / 1601 |
| `tc_supported` | the tensor-core route | D % 4 == 0, D <= 1024 |

Plus a source lint: every kernel with dynamic shared memory opts in to its size with cudaFuncSetAttribute, and every
one whose dynamic buffer holds feature rows also has a route for rows that do not fit (global memory, or a feature cap
its launcher enforces)."""
import importlib.util
import os
import re

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "kmcuda_b200", "csrc")
DEFAULT_DYNAMIC_SMEM = 48 * 1024
MAX_D = 65535


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _constant(name, fname):
    m = re.search(r"constexpr\s+\w+\s+%s\s*=\s*([^;]+);" % name, _src(fname))
    assert m, (name, fname)
    return int(eval(m.group(1).replace("sizeof(float)", "4")))


@pytest.fixture(scope="module")
def gpu_module():
    spec = importlib.util.spec_from_file_location("test_exact_route_gpu", os.path.join(HERE, "test_exact_route_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# ---------------------------------------------------------------------------------------------- the switches
def exact_cfg(D):
    """simt_kernels.cu::exact_cfg: (rows per CTA, shared memory staging)"""
    src = _src("simt_kernels.cu")
    body = src[src.index("static ExactCfg exact_cfg(int D)"):]
    body = body[:body.index("\n}\n")]
    assert "const size_t limit = 200 * 1024;" in body and "for (int rb : {128, 64, 32})" in body
    assert "int tpr = 1024 / rb > 8 ? 8 : 1024 / rb;" in body
    assert "static_cast<size_t>(rb + 1) * D * sizeof(float) + static_cast<size_t>(tpr) * rb * 8" in body
    assert "return {128, 8, 0," in body
    for rb in (128, 64, 32):
        tpr = min(8, 1024 // rb)
        if (rb + 1) * D * 4 + tpr * rb * 8 <= 200 * 1024:
            return rb, True
    return 128, False


def _row_limits():
    """(largest D that launched without opting in, kRowStageMaxD) of the two one-CTA-per-row kernels"""
    out = {}
    for kernel, fname in (("exact_rows_few_kernel", "simt_kernels.cu"), ("yy_rows_cta_kernel", "yinyang.cu")):
        src = _src(fname)
        body = src[src.index(kernel + "("):]
        body = body[:body.index("\n}\n")]
        static = 0
        for decl in re.findall(r"__shared__\s+(?:float|uint32_t)\s+([^;]+);", body):
            static += sum(4 * int(n) for n in re.findall(r"\[(\d+)\]", decl))
        out[kernel] = static
    assert out == {"exact_rows_few_kernel": 4096, "yy_rows_cta_kernel": 4096}, out
    return (DEFAULT_DYNAMIC_SMEM - 4096) // 4, _constant("kRowStageMaxD", "kernels.h")


def test_restated_switches_match_the_sources():
    assert [D for D in range(1, 2000) if exact_cfg(D) != exact_cfg(D + 1)] == [381, 771, 1536]
    assert exact_cfg(1536) == (32, True) and exact_cfg(1537) == (128, False) and exact_cfg(MAX_D) == (128, False)
    assert _constant("kFewRows", "simt_kernels.cu") == 8192
    assert _constant("kKnnMaxSmemD", "knn_kernels.cu") == 2048
    assert _row_limits() == (11264, 16384)
    assert _constant("kStrictMaxD", "kernels.h") == 1600
    # the launchers use these constants
    assert "D <= kRowStageMaxD ? D : 0" in _src("simt_kernels.cu") and "D <= kRowStageMaxD ? D : 0" in _src("yinyang.cu")
    assert "D <= kKnnMaxSmemD ? D : 0" in _src("knn_kernels.cu")
    assert "if (D > kStrictMaxD) return cudaErrorInvalidValue;" in _src("simt_kernels.cu")
    assert "> kStrictMaxD" in _src("api.cu")
    tc = _src("assign_tc.cu")
    assert "if (D < 4 || D % 4 != 0 || D > tc::MAX_TILE64_NKB * tc::KB) return false;" in tc


def test_gpu_helpers_match_the_restatement(gpu_module):
    for D in list(range(1, 4100)) + [11264, 11265, 12287, 16384, 16385, MAX_D]:
        assert gpu_module.tile_rows(D) == exact_cfg(D)[0], D
        assert gpu_module.tc_shape(D) == (D >= 4 and D % 4 == 0 and D <= 1024), D


def _straddles(values, boundary):
    return boundary in values and boundary + 1 in values


def test_shape_lists_straddle_every_switch(gpu_module):
    g = gpu_module
    lloyd = set(g.LLOYD_D) | set(g.LLOYD_WIDE_D)
    tiers = [D for D in range(1, MAX_D) if exact_cfg(D) != exact_cfg(D + 1)]
    few = _constant("kFewRows", "simt_kernels.cu")
    knn = _constant("kKnnMaxSmemD", "knn_kernels.cu")
    default_row, stage_row = _row_limits()
    strict = _constant("kStrictMaxD", "kernels.h")
    for b in tiers:
        assert _straddles(lloyd, b), ("Lloyd pass", b)
        assert {D for D in g.REFRESH_D if exact_cfg(D)[0] == exact_cfg(b)[0]}, ("refresh", b)
    assert _straddles(g.LIST_LENGTHS, few) and 1 in g.LIST_LENGTHS
    assert _straddles(g.KNN_D, knn)
    for b in (default_row, stage_row):
        assert _straddles(g.LIST_D, b), ("row lists", b)
        assert _straddles(g.YY_D, b), ("Yinyang rows", b)
    assert _straddles(lloyd, default_row)
    assert g.STRICT_D[-1] == strict and g.STRICT_REJECTED_D == strict + 1
    assert _straddles(g.STRICT_D, 1536)                             # the strict runs cross the exact pass's last tier
    # just past the tensor-core envelope, D % 4 != 0 on every tier, and the largest D the API accepts
    assert {1025, 1026, 1028} <= lloyd and {1, 3, 5, 33, 126} <= lloyd and MAX_D in lloyd
    assert {12287, MAX_D} <= set(g.ACCEPT_D) and any(D > default_row for D in g.EXT_D)
    # the member sums: VEC 1 (D % 4 != 0, unaligned X), VEC 4 with more float4 columns than the CTA has threads
    assert any(D % 4 for D, _, _ in g.SUMS) and any(u for _, _, u in g.SUMS)
    assert any(D % 4 == 0 and D // 4 > 256 and not u for D, _, u in g.SUMS)
    # k-NN list chunks of 32 entries: k below, at and above one and two chunks
    assert {1, 31, 32, 33, 65} <= set(g.KNN_K)
    # fp16x2 with an odd count of packed pairs
    assert g.FP16_D % 4 == 2 and not g.tc_shape(g.FP16_D)
    # every shape runs on the exact route except the one forced there (inside the tensor-core envelope)
    all_d = lloyd | set(g.LIST_D) | set(g.REFRESH_D) | set(g.YY_D) | set(g.STRICT_D) | set(g.AVG_D) | set(g.KNN_D) | \
        set(g.EXT_D) | set(g.ACCEPT_D) | {g.FP16_D}
    assert {D for D in all_d if g.tc_shape(D)} == {772}
    assert 772 not in g.YY_D and 772 not in g.STRICT_D


# ---------------------------------------------------------------------------------------------- dynamic shared memory
def _kernels_with_dynamic_smem():
    """{kernel name: (file, parameter list)} of every kernel that declares extern __shared__, itself or in a device
    function it calls (the tensor-core kernels)"""
    out = {}
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith((".cu", ".cuh")):
            continue
        src = _src(name)
        heads = []
        for m in re.finditer(r"(__global__\s+|__device__[^;{(]*?)void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*"
                             r"\(([^{;]*?)\)\s*\{", src):
            body = src[m.end():src.index("\n}\n", m.end())]
            heads.append((m.start(), m.group(2), m.group(3), m.group(1).startswith("__global__"), body))
        for m in re.finditer(r"extern\s+__shared__", src):
            owner = [h for h in heads if h[0] < m.start()][-1]
            callers = [owner] if owner[3] else \
                [h for h in heads if h[3] and re.search(r"\b%s\s*[<(]" % owner[1], h[4])]
            assert callers, owner[1]
            out.update({h[1]: (name, h[2]) for h in callers})
    return out


def _opted_in(kernel, fname):
    """the file calls cudaFuncSetAttribute(MaxDynamicSharedMemorySize) on the kernel, directly or through a variable
    bound to it"""
    src = _src(fname)
    names = {kernel}
    for m in re.finditer(r"auto\s+(\w+)\s*=\s*([^;]+);", src):
        if re.search(r"\b%s\b" % kernel, m.group(2)):
            names.add(m.group(1))
    for m in re.finditer(r"cudaFuncSetAttribute\(\s*([^;]+?),\s*cudaFuncAttributeMaxDynamicSharedMemorySize", src):
        if any(re.search(r"\b%s\b" % n, m.group(1)) for n in names):
            return True
    return False


def test_dynamic_shared_memory_kernels_opt_in_and_have_a_route_for_wide_rows():
    kernels = _kernels_with_dynamic_smem()
    assert {"exact_pass_kernel", "exact_rows_few_kernel", "yy_rows_cta_kernel", "knn_warp_search_kernel",
            "strict_adjust_kernel", "tc_assign_kernel", "tc_assign_rows_kernel"} <= set(kernels), kernels
    for kernel, (fname, params) in kernels.items():
        assert _opted_in(kernel, fname), "%s (%s) launches with dynamic shared memory without opting in" % (kernel, fname)
        if re.search(r"\bint\s+D\b", params):
            # the buffer holds feature rows: a switch to global memory, or a cap the launcher enforces
            capped = kernel == "strict_adjust_kernel" and "if (D > kStrictMaxD) return" in _src(fname)
            assert re.search(r"\bint\s+(use_smem|smem_d)\b", params) or capped, \
                "%s (%s) has no route for rows that do not fit in shared memory" % (kernel, fname)
