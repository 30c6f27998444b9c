"""The Philox4x32-10 dropout reference (oracle/philox.py) without a GPU: Random123 known answers, a cross-check against cuRAND's
own host-compiled curand_Philox4x32_10, the case table of tests/test_dropout_exact_gpu.py, and negative controls: each
realistic bug of the mask mapping changes the mask on that file's own cases."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import bf16_split as S
from oracle import philox as PH
from tests.test_dropout_exact_gpu import GRID_CAP_N, KEEPS, SEEDS, SIMT_CASES, STREAMS, TC_CASES
from tests.test_tc_split_exact_gpu import expected_ksplit

KAT = [  # Random123 kat_vectors, philox4x32 10 rounds: (ctr, key, output)
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]

# what each GPU case reaches: (entry point, path / tile)
CASE_MAP = {
    "apply_matrix": ("pnp_dropout_apply", "float4 body + scalar tail (n = 4099), every seed x stream x keep"),
    "apply_tails": ("pnp_dropout_apply", "scalar tail only and after whole quads, n & 3 = 0 .. 3"),
    "apply_grid_cap": ("pnp_dropout_apply", "grid-stride loop past the 8448-CTA cap, in place"),
    "apply_disabled": ("pnp_dropout_apply", "NULL seed / keep 1 / no cfg: copy, out of place and in place"),
    "float4_C16": ("pnp_conv2d_fwd", "float4 store, accumulate"),
    "scalar_C6": ("pnp_conv2d_fwd", "scalar store (Cout % 4 = 2), accumulate"),
    "scalar_C5": ("pnp_conv2d_fwd", "scalar store (Cout % 4 = 1), accumulate"),
    "n16_72wide": ("pnp_conv2d_tc_fwd / _fused", "BLOCK_N 16, unused tile rows"),
    "n32": ("pnp_conv2d_tc_fwd / _fused", "BLOCK_N 32"),
    "n64_ragged": ("pnp_conv2d_tc_fwd / _fused", "BLOCK_N 64, ragged last tile"),
    "n128": ("pnp_conv2d_tc_fwd / _fused", "BLOCK_N 128"),
    "n128_8imgs_per_tile": ("pnp_conv2d_tc_fwd / _fused", "BLOCK_N 128, 8 images per tile, ragged last tile"),
    "splitk": ("pnp_conv2d_tc_fwd", "BLOCK_N 64, split-K (atomic partials times the mask)"),
    "bn_bwd": ("pnp_bn_bwd_apply, pnp_bn_bwd_apply_fused, pnp_bn_bwd_apply_direct",
               "test_elementwise_exact_gpu.py::test_bn_bwd_apply_exact through drop_mask"),
    "seed_sequence": ("pnp_seed_advance -> pnp_dropout_apply / pnp_conv2d_fwd / pnp_conv2d_tc_fwd", "stream order, and PNP_PDL=1"),
    "graph": ("pnp_seed_advance + pnp_dropout_apply", "captured CUDA graph, 3 replays"),
}
PRODUCERS = {"pnp_dropout_apply", "pnp_conv2d_fwd", "pnp_conv2d_tc_fwd", "pnp_conv2d_tc_fwd / _fused", "pnp_bn_bwd_apply",
             "pnp_bn_bwd_apply_fused", "pnp_bn_bwd_apply_direct"}


def test_known_answers():
    for ctr, key, out in KAT:
        assert tuple(int(v) for v in PH.philox4x32_10(ctr, key)) == out


def test_matches_curand(tmp_path):
    """4096 deterministic (ctr, key) pairs through cuRAND's curand_Philox4x32_10, compiled for the host"""
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = tmp_path / "philox_host.cu"
    src.write_text(
        "#define QUALIFIERS static inline __host__ __device__\n"
        "#include <cstdio>\n#include <cuda_runtime.h>\n#include <curand_philox4x32_x.h>\n"
        "int main() {\n  unsigned c0, c1, c2, c3, k0, k1;\n"
        "  while (scanf(\"%x %x %x %x %x %x\", &c0, &c1, &c2, &c3, &k0, &k1) == 6) {\n"
        "    uint4 r = curand_Philox4x32_10(make_uint4(c0, c1, c2, c3), make_uint2(k0, k1));\n"
        "    printf(\"%08x %08x %08x %08x\\n\", r.x, r.y, r.z, r.w);\n  }\n  return 0;\n}\n")
    exe = tmp_path / "philox_host"
    subprocess.run([nvcc, "-o", str(exe), str(src)], check=True, capture_output=True, timeout=300)
    rng = np.random.default_rng(2024)
    words = rng.integers(0, 1 << 32, size=(4096, 6), dtype=np.uint64)
    words[:64, :4] = np.arange(64)[:, None]               # small counters, as dropout draws them
    words[64:128] = 0xFFFFFFFF - np.arange(64)[:, None]    # the wrap-around end
    inp = "\n".join(" ".join("%x" % int(v) for v in row) for row in words)
    out = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True, timeout=60).stdout.split()
    want = np.array([int(v, 16) for v in out], dtype=np.uint64).reshape(-1, 4)
    got = PH.philox4x32_10(words[:, :4], words[:, 4:]).astype(np.uint64)
    assert want.shape == got.shape and np.array_equal(want, got)


def test_threshold_and_multiplier():
    assert PH.keep_threshold(0.5) == 32768 and PH.keep_threshold(0.75) == 49152
    assert PH.keep_threshold(0.3) == 19661            # 19660.8 + 0.5: the rounding decides
    assert PH.keep_threshold(2.0 ** -16) == 1 and PH.keep_threshold(1 - 2.0 ** -16) == 65535
    assert PH.keep_threshold(0.99999) == 65535 and PH.keep_threshold(1.0) == 65536 and PH.keep_threshold(0.0) == 0
    assert PH.inv_keep(0.75) == np.float32(1.0) / np.float32(0.75)
    assert np.all(PH.dropout_mult(None, 3, 0.5, 17) == 1) and np.all(PH.dropout_mult(5, 3, 1.0, 17) == 1)


def test_seed_advance_wraps():
    assert PH.seed_advance(0) == PH.LCG_INC
    s = (1 << 64) - 1
    assert PH.seed_advance(s) == (s * PH.LCG_MUL + PH.LCG_INC) % (1 << 64)
    assert PH.seed_advance(s, 3) == PH.seed_advance(PH.seed_advance(PH.seed_advance(s)))


def test_kept_fraction_is_binomial():
    n = 1 << 20
    for keep in (0.5, 0.3, 0.6137):
        f = float((PH.dropout_mult(0x5EED, 7, keep, n) != 0).mean())
        assert abs(f - PH.keep_threshold(keep) / 65536) < 5 * np.sqrt(keep * (1 - keep) / n), (keep, f)


def test_case_table_reaches_every_producer_and_tile():
    from tests import test_dropout_exact_gpu as G
    ids = {c[0] for c in SIMT_CASES} | {c[0] for c in TC_CASES}
    assert ids <= set(CASE_MAP), ids - set(CASE_MAP)
    reached = set()
    for entry, _ in CASE_MAP.values():
        reached |= {e.strip() for e in entry.replace("->", ",").split(",")}
    assert PRODUCERS <= reached, PRODUCERS - reached
    assert {c[7] for c in TC_CASES} == {16, 32, 64, 128}
    assert any(c[5] % 4 == 0 for c in SIMT_CASES) and any(c[5] % 4 for c in SIMT_CASES)
    assert GRID_CAP_N > 4 * 8448 * 1024 and hasattr(G, "test_exact_cases_under_pdl")
    for tag, B, H, W, Cin, Cout, keep, block_n, split in TC_CASES:
        g = S.Geom(B, H, W, Cin, H, W, Cout, 3, 3, 1, 1, 1, 1)
        assert (Cout % 128 == 0 and block_n == 128) or block_n == Cout, tag
        assert (expected_ksplit("fwd", g, 132) > 1) == split, tag
        if split:      # a split-K partial times 1/keep must be exact
            assert float(PH.inv_keep(keep)) in (2.0, 4.0, 65536.0), tag


# ------------------------------------------------------------------------------------------------
# negative controls
# ------------------------------------------------------------------------------------------------
def mutant_mult(seed, stream, keep, n, mutation):
    """dropout_mult with one realistic bug"""
    i = np.arange(n, dtype=np.int64)
    per = 4 if mutation == "block_per_4" else 8
    nb = (n + per - 1) // per
    b = np.arange(nb, dtype=np.uint64)
    m32 = np.uint64(0xFFFFFFFF)
    ctr = [b & m32, b >> np.uint64(32), np.full_like(b, PH.lo32(stream)), np.full_like(b, PH.hi32(stream))]
    key = [np.full_like(b, PH.lo32(seed)), np.full_like(b, PH.hi32(seed))]
    if mutation == "stream_hi_dropped":
        ctr[3] = np.zeros_like(b)
    if mutation == "seed_hi_dropped":
        key[1] = np.zeros_like(b)
    if mutation == "ctr_key_swapped":
        ctr, key = key + ctr[2:], ctr[:2]
    words = PH.philox4x32_10(np.stack(ctr, -1), np.stack(key, -1)).reshape(-1)
    if mutation == "quad_half_ignored":
        w = words[4 * (i >> 3) + ((i & 3) >> 1)]
    elif mutation == "block_per_4":
        w = words[4 * (i >> 2) + ((i & 3) >> 1)]
    else:
        w = words[4 * (i >> 3) + ((i & 7) >> 1)]
    odd = (i & 1) == 1
    if mutation == "halves_swapped":
        odd = ~odd
    u = np.where(odd, w >> np.uint32(16), w & np.uint32(0xFFFF)).astype(np.int64)
    t = PH.keep_threshold(keep)
    if mutation == "no_half_rounding":
        t = int(np.float32(np.float32(keep) * np.float32(65536.0)))
    kept = u <= t if mutation == "le_threshold" else u < t
    return np.where(kept, PH.inv_keep(keep), np.float32(0)).astype(np.float32)


MUTATIONS = ["ctr_key_swapped", "stream_hi_dropped", "seed_hi_dropped", "halves_swapped", "quad_half_ignored", "no_half_rounding",
             "le_threshold", "block_per_4"]


def test_mutant_helper_is_the_reference_without_a_mutation():
    for seed, stream, keep in ((SEEDS[3], STREAMS[3], 0.3), (SEEDS[1], STREAMS[4], 0.75)):
        assert np.array_equal(mutant_mult(seed, stream, keep, 4099, None), PH.dropout_mult(seed, stream, keep, 4099))


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutations_change_the_mask_on_the_gpu_cases(mutation):
    """over the pnp_dropout_apply matrix of the GPU file (n = 4099), count the elements and cases the bug changes"""
    elements, cases = 0, 0
    for keep in KEEPS:
        for seed in SEEDS:
            for stream in STREAMS:
                d = int((mutant_mult(seed, stream, keep, 4099, mutation) != PH.dropout_mult(seed, stream, keep, 4099)).sum())
                elements += d
                cases += d > 0
    print("  %-18s changes %7d elements in %3d of %d cases" % (mutation, elements, cases, len(KEEPS) * len(SEEDS) * len(STREAMS)))
    assert elements > 0
