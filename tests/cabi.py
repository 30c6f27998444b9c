"""The kernel-level harness of the C-ABI tests: the library handle, device pointers, seeded operand draws, NaN-sentinel buffers
and the check that a rejected call left its buffers alone, the bf16 operand planes, the dropout configuration, the wgmma
launchers' tile and split-K rule, and re-runs of a test file's cases in a child process under a launch-mode switch.

It imports without a GPU: pnp_b200 is imported inside lib()."""
import ctypes
import os
import re
import subprocess
import sys
import time

import pytest
import torch

from oracle import bf16_split as S
from oracle import philox

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
BAD_ARG, UNSUPPORTED = 100001, 100002
SENTINEL = 0x7FC0BEEF           # a quiet NaN no kernel computes


def lib(require_tc=False):
    """-> (_C, runtime) of the built library; require_tc: fail where the wgmma path is unavailable (it is the one H100 runs)"""
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C, runtime as rt
    if require_tc and not rt.tc_available():
        pytest.fail("wgmma path unavailable on this device -- it must be the one that runs on H100")
    return _C, rt


def ptr(t):
    return None if t is None else t.data_ptr()


def sync():
    torch.cuda.synchronize()


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ------------------------------------------------------------------------------------------------
# seeded operands: a CPU generator draws on the host, a CUDA generator on the device (the two streams differ)
# ------------------------------------------------------------------------------------------------
def cpu_gen(seed):
    return torch.Generator().manual_seed(seed)


def dev_gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def ints(shape, lo, hi, gen, scale=1.0):
    """uniform integers in [lo, hi] as fp32, times scale, on the generator's device"""
    return torch.randint(lo, hi + 1, shape, generator=gen, device=gen.device).float() * scale


def pick(shape, values, gen):
    """elements drawn uniformly from `values` (fp32), on the generator's device"""
    v = torch.tensor(values, dtype=torch.float32, device=gen.device)
    return v[torch.randint(0, len(values), shape, generator=gen, device=gen.device)]


# ------------------------------------------------------------------------------------------------
# bit patterns and rejected calls
# ------------------------------------------------------------------------------------------------
def sentinel(shape, dev=DEV):
    return torch.full(shape if isinstance(shape, tuple) else (shape,), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)


def assert_bits(tag, got, ref):
    g = got.contiguous().view(torch.int32).reshape(-1)
    r = ref.float().contiguous().view(torch.int32).reshape(-1)
    assert g.shape == r.shape, (tag, tuple(got.shape), tuple(ref.shape))
    bad = (g != r).nonzero()
    if bad.numel():
        i = int(bad[0])
        raise AssertionError("%s: %d of %d elements differ; first at flat %d: got %r (0x%08x), ref %r (0x%08x)" % (
            tag, bad.numel(), g.numel(), i, float(got.reshape(-1)[i]), int(g[i]) & 0xFFFFFFFF, float(ref.reshape(-1)[i]),
            int(r[i]) & 0xFFFFFFFF))


def snapshot(bufs):
    """copies of the buffers a call must leave untouched (None entries are skipped)"""
    return {k: t.clone() for k, t in bufs.items() if t is not None}


def assert_untouched(tag, name, bufs, before):
    """every buffer still holds the bytes of its snapshot (NaN sentinels, fp64 fills and labels alike); a buffer the call
    was given as NULL is skipped"""
    sync()
    for k, t in before.items():
        if bufs[k] is not None:
            assert torch.equal(bufs[k].view(torch.uint8), t.view(torch.uint8)), "%s: %s wrote %s" % (tag, name, k)


# ------------------------------------------------------------------------------------------------
# bf16 operand planes
# ------------------------------------------------------------------------------------------------
def empty_planes(shape, nterms):
    """uninitialised (hi, lo) bf16 planes; lo only at nterms 3"""
    hi = torch.empty(shape, dtype=torch.bfloat16, device=DEV)
    return hi, (torch.empty(shape, dtype=torch.bfloat16, device=DEV) if nterms == 3 else None)


def split_dev(_C, rt, x, nterms):
    """(hi, lo) planes of the fp32 activations x by pnp_split_bf16"""
    hi, lo = empty_planes(x.shape, nterms)
    _C.call("pnp_split_bf16", _C.ptr(x), _C.ptr(hi), _C.ptr(lo), x.numel(), rt.stream())
    return hi, lo


def split_w_dev(_C, rt, w, for_dgrad, nterms, cin_pad=0):
    """(hi, lo) planes of the HWIO weights w by pnp_split_weight_bf16, in the forward or the data-gradient layout"""
    kh, kw, cin, cout = w.shape
    hi, lo = empty_planes((kh * kw * max(cin, cin_pad) * cout,), nterms)
    _C.call("pnp_split_weight_bf16", _C.ptr(w), _C.ptr(hi), _C.ptr(lo), kh, kw, cin, cout, 1 if for_dgrad else 0, cin_pad,
            rt.stream())
    return hi, lo


def assert_planes(tag, hi, lo, fp32):
    rh, rl = S.split(fp32.cpu())
    assert S.planes_equal(hi.cpu().reshape(rh.shape), rh), "%s: hi plane is not rn_bf16(x)" % tag
    if lo is not None:
        assert S.planes_equal(lo.cpu().reshape(rl.shape), rl), "%s: lo plane is not rn_bf16(x - hi)" % tag


# ------------------------------------------------------------------------------------------------
# dropout
# ------------------------------------------------------------------------------------------------
def drop_cfg(_C, keep, stream_id=11, seed=0x1234_5678_9ABC):
    """-> (DropCfg, its device seed tensor, which must outlive every launch that reads it)"""
    seed_t = torch.tensor([seed], dtype=torch.int64, device=DEV)
    cfg = _C.DropCfg(seed_t.data_ptr(), stream_id, keep)
    cfg.seed_value = seed
    return cfg, seed_t


def drop_mask(cfg, shape):
    """the multipliers of (seed, stream, keep) from the independent Philox4x32-10 reference (oracle/philox.py)"""
    n = 1
    for s in shape:
        n *= int(s)
    m = philox.dropout_mult(cfg.seed_value, cfg.stream, cfg.keep, n)
    return torch.from_numpy(m).reshape(tuple(shape)).to(DEV)


# ------------------------------------------------------------------------------------------------
# the wgmma launchers' tile rule (conv_tc.cu choose_tile / run_tc)
# ------------------------------------------------------------------------------------------------
def cdiv(a, b):
    return -(-a // b)


def same_pad(n, k, s, d=1):
    out = -(-n // s)
    total = max((out - 1) * s + (k - 1) * d + 1 - n, 0)
    return total // 2


def last_config(_C):
    """(BLOCK_N, BLOCK_K, split-K factor) of the last wgmma launch"""
    n_, k_, s_ = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
    _C.lib.pnp_tc_last_config(ctypes.byref(n_), ctypes.byref(k_), ctypes.byref(s_))
    return n_.value, k_.value, s_.value


def block_n(N):
    """accumulator tile width for N output columns"""
    return 128 if N % 128 == 0 else (64 if N % 64 == 0 else (32 if N % 32 == 0 else 16))


def choose_tile(U, V, B):
    """pixel tile (tw, th, tn) of 128 output pixels over a U x V grid (choose_tile, exact = 0)"""
    if V >= 128:
        return 128, 1, 1
    tw, th = V, min(128 // V, U)
    tn = max(128 // (tw * th), 1) if th == U else 1
    return tw, th, min(tn, B)


def k_block(n_cols, K):
    bk = 64 if K % 64 == 0 else (32 if K % 32 == 0 else 16)
    if bk == 64 and n_cols in (128, 64) and os.environ.get("PNP_TC_BK%d" % n_cols, "64").strip() == "32":
        bk = 32
    return bk


def fwd_tiles(g):
    """(m-tiles, n-tiles) of the forward launcher on a stride-1 geometry"""
    tw, th, tn = choose_tile(g.Ho, g.Wo, g.B)
    return cdiv(g.Wo, tw) * cdiv(g.Ho, th) * cdiv(g.B, tn), g.Cout // block_n(g.Cout)


def crosses_ntile(g, sms):
    """does some persistent CTA walk tiles of two different n-tiles (tile t -> n-tile t % n_tiles, CTA b walks b, b + sms, ..)"""
    mt, nt = fwd_tiles(g)
    total = mt * nt
    return any(len({t % nt for t in range(b, total, sms)}) > 1 for b in range(min(sms, total)))


def expected_ksplit(launcher, g, sms):
    """split-K factor the forward / data-gradient launcher picks for geometry g (no fused epilogue) on a device with `sms`
    SMs: split when the layer has at most half as many tiles as SMs and at least 8 k-blocks in its shallowest phase, by
    min(sms / tiles, k-blocks / 4, 32)"""
    if launcher == "fwd":
        N, K = g.Cout, g.Cin
        phases = [(g.Ho, g.Wo, g.kh * g.kw)]
    else:
        N, K, s = g.Cin, g.Cout, g.stride
        phases = []
        for py in range(s):
            for px in range(s):
                Up, Vp = (g.H - py + s - 1) // s, (g.W - px + s - 1) // s
                if Up <= 0 or Vp <= 0:
                    continue
                ty = sum(1 for k in range(g.kh) if (py + g.pad_t - k * g.dil) % s == 0)
                tx = sum(1 for k in range(g.kw) if (px + g.pad_l - k * g.dil) % s == 0)
                phases.append((Up, Vp, ty * tx))
    U, V = max(p[0] for p in phases), max(p[1] for p in phases)
    tw, th, tn = choose_tile(U, V, g.B)
    n_cols = block_n(N)
    kchunks = K // k_block(n_cols, K)
    tiles = sum(cdiv(Vp, tw) * cdiv(Up, th) for Up, Vp, _ in phases) * cdiv(g.B, tn) * (N // n_cols)
    min_kb = min(t for _, _, t in phases) * kchunks
    if tiles * 2 > sms or min_kb < 8:
        return 1
    return max(1, min(sms // tiles, min_kb // 4, 32))


# ------------------------------------------------------------------------------------------------
# launch-mode switches are read once per process: their cases re-run in a child
# ------------------------------------------------------------------------------------------------
def rerun(env, file, selection, flags=(), timeout=280):
    """pytest -q -x -p no:cacheprovider <file> -k <selection> in a child process with `env` added to the environment; prints
    the child's summary line and wall time, fails unless it passed, -> (tests passed, its output lines)"""
    t0 = time.time()
    p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", *flags, "-p", "no:cacheprovider", os.path.join(ROOT, file),
                        "-k", selection], cwd=ROOT, env=dict(os.environ, **env), capture_output=True, text=True, timeout=timeout)
    lines = p.stdout.splitlines()
    print("  %s: %s (wall %.1f s)" % (" ".join("%s=%s" % kv for kv in env.items()), lines[-1] if lines else "", time.time() - t0))
    assert p.returncode == 0, "\n".join(lines[-25:])
    m = re.search(r"(\d+) passed", lines[-1])
    return (int(m.group(1)) if m else 0), lines
