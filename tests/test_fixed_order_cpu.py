"""The deterministic building blocks of the seeding, mini-batch, relocation and restart kernels live once, in
csrc/fixed_order.cuh (hash, unit conversions, mass, block partial, 1024-chunk fold) and exact.cuh (the staged slice
load).  Their promises -- draws independent of the device split and launch shape, sums added in one fixed order --
hold only while every kernel calls the same code, so a second copy in kmcuda_b200/csrc is a failure here."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kmcuda_b200", "csrc")


def sources():
    out = {}
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".h", ".cc")):
            with open(os.path.join(CSRC, f)) as fh:
                out[f] = fh.read()
    return out


def files_matching(pattern):
    rx = re.compile(pattern)
    return sorted(f for f, s in sources().items() if rx.search(s))


@pytest.mark.parametrize("const", ["0x9E3779B97F4A7C15", "0xBF58476D1CE4E5B9", "0x94D049BB133111EB"])
def test_splitmix64_constants_in_one_file(const):
    assert files_matching(re.escape(const)) == ["fixed_order.cuh"]


def test_one_splitmix64_definition():
    defs = [(f, m) for f, s in sources().items() for m in re.findall(r"uint64_t\s+(\w+)\s*\(uint64_t z\)", s)]
    assert defs == [("fixed_order.cuh", "splitmix64")]


def test_cdiv_defined_once():
    rx = r"(?:inline|static)[^;{]*\bunsigned\s+\w+\s*\(size_t a, size_t b\)"
    assert files_matching(rx) == ["kernels.h"]
    assert len(re.findall(rx, sources()["kernels.h"])) == 1


def test_unit_conversions_only_in_helpers():
    # h >> 11 scaled by 2^-53: the two 53-bit unit conversions of the counter hash (seeding.cu's is the host
    # AFK-MC2 sampler's draw from std::mt19937_64, another generator)
    assert files_matching(r"9007199254740992") == ["fixed_order.cuh", "seeding.cu"]


def test_chunk_fold_only_in_helpers():
    # the per-thread chunk of ceil(n / 1024) terms and the sequential fold of the 1024 chunk sums
    assert files_matching(r"\+ 1023\) / 1024") == ["fixed_order.cuh"]
    assert files_matching(r"for \(int q = 0; q < 1024; q\+\+\)") == ["fixed_order.cuh"]


def test_block_partial_only_in_helper():
    # thread 0 adding the per-warp double partials in order
    assert files_matching(r"/ 32; \w+\+\+\) \w+ \+= s_part\[") == ["fixed_order.cuh"]


def test_staged_tile_load_only_in_stager():
    # the padded 33-float row stride of the 32-feature slice written from X
    assert files_matching(r"tile\[r \* 33 \+ lane\] = \(") == ["exact.cuh"]
    assert len(re.findall(r"tile\[r \* 33 \+ lane\] = \(", sources()["exact.cuh"])) == 1


@pytest.mark.parametrize("name", ["kmp_mix", "gpp_mix", "mb_mix", "mb_unit", "kmp_mass", "gpp_mass", "cdivk",
                                  "kmp_sum_kernel", "launch_kmp_sum"])
def test_removed_names_are_gone(name):
    assert files_matching(r"\b%s\b" % name) == []


def test_one_eligibility_rule_for_keys_and_inertia():
    s = sources()["relocate.cu"]
    assert len(re.findall(r"a < K && wi > 0\.f", s)) == 1
    for kernel in ("reloc_keys_kernel", "inertia_kernel"):
        body = s.split(kernel + "(const float*")[1].split("\n}\n")[0]
        assert "eligible_own_distance<VEC4, METRIC>(" in body, kernel
