"""Both attention kernels element by element against float64, with error bounds derived from their rounding points.

lseg_mhsa (csrc/mhsa.cuh, the wgmma flash attention of every ViT block) is compared with softmax(0.125 q k^T [+ causal
mask]) v evaluated in float64 from the same fp16 q, k and v. Every output element must lie within the bound that
tests/attention_oracle.py derives from the kernel's own rounding points (fp32 S on the tensor cores, ex2 or exp2_poly<3>,
P rounded to fp16, fp32 PV and l, the final fp16 rounding; the derivation is that module's docstring). The input
families are chosen so that a wrong key count, a misplaced key tile, a missed rescale or a wrong causal diagonal moves
some element far outside that bound:
  flat     q = 0, v small integers: every output is exactly sum(v) / n_visible, checked to 0.5 ulp + 2^-22 + eps_exp
           relative: pins the key count of every row (tails, tile boundaries, the causal diagonal);
  planted  rows whose one-hot q channel matches one key only, 12.5 nats above the rest, at keys 0, 63, 64, 127, 128,
           N-1 and (causal) the diagonal: the output is that key's v row, so a misplaced K/V tile shows;
  rising   scores rise with the key index: the running maximum moves in every 64-key tile (the O / l rescale);
  falling  the maximum sits in the first tile and later tiles underflow;
  wide     a score range above 150 in log2 units, past the -126 clamp of the POLY path;
  random1, random3   randn at amplitude 1 and 3 (seed 19: the inputs of tests/test_ops_gpu.py::test_mhsa, on every shape here).
Every output lives between guard rows of a NaN sentinel that must keep its bits, qkv must be unchanged, each image
computed alone must equal its rows of the batch bit for bit, and a second run must repeat the first.

lseg_text_attn (csrc/text_attn.cuh, the CLIP text tower) is compared with an emulation of its rounding points in float32
in the kernel's order (attention_oracle.text_attn_emulate): within 1 fp16 ulp everywhere and bit-identical on nearly
all elements (only expf can differ); with q = 0 the emulation is exact and the kernel must match it bit for bit.
"""
import os

import pytest
import torch

from attention_oracle import (EPS_EX2, EPS_POLY, MHSA_SHAPES, flat_reference, flat_tolerance, mhsa_oracle,
                              text_attn_emulate, text_attn_flat, ulp16, violations)

pytestmark = pytest.mark.gpu

SENT = 0x7E5A  # fp16 NaN
GUARD = 64     # sentinel rows before and after every output


@pytest.fixture(scope="module")
def ops():
    import lseg_b200  # noqa: F401
    from lseg_b200 import ops as _ops
    return _ops


@pytest.fixture(autouse=True)
def _watchdog(ops):
    yield
    torch.cuda.synchronize()
    wd = ops.read_watchdog()
    assert wd[0] == 0, f"device barrier watchdog fired: tag={wd[0]} block={wd[1]} thread={wd[2]} parity={wd[3]}"


def _guarded(rows, cols):
    """Flat fp16 buffer: GUARD sentinel rows, the [rows, cols] output, GUARD sentinel rows. Returns (buffer, output)."""
    buf = torch.full(((rows + 2 * GUARD) * cols,), SENT, dtype=torch.int16, device="cuda").view(torch.float16)
    return buf, buf[GUARD * cols:(GUARD + rows) * cols].view(rows, cols)


def _guards_intact(buf, rows, cols, what):
    b = buf.view(torch.int16)
    outside = torch.cat([b[:GUARD * cols], b[(GUARD + rows) * cols:]])
    n = int((outside != SENT).sum())
    assert n == 0, f"{what}: {n} elements of the guard rows were written"


def _same_bits(a, b, what):
    bad = a.view(torch.int16) != b.view(torch.int16)
    n = int(bad.sum())
    if n:
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {n} elements differ; first at {i}: {a[tuple(i)].item()} vs {b[tuple(i)].item()}")


def _env_variant():
    return int(os.environ.get("LSEG_MHSA_VARIANT", "0"))


def _eps_exp(variant):
    """MUFU ex2 only (instantiation 0) or part of the exponentials on exp2_poly<3> (3, 7 and 4, 8)."""
    v = _env_variant() if variant is None else variant
    return EPS_POLY if v in (3, 4, 7, 8) else EPS_EX2


# ---------------------------------------------------------------------------------------------------------------------
# lseg_mhsa
# ---------------------------------------------------------------------------------------------------------------------
_HEADS = [1, 2, 3, 12, 16]
EDGE_SHAPES = [(1 + i % 2, n, _HEADS[(i + 2 * c) % 5], bool(c))
               for i, n in enumerate([1, 2, 63, 127, 128, 129, 191, 192, 255, 256, 257]) for c in (0, 1)]
ENGINE_SHAPES = [(8, 901, 16, False), (4, 2117, 16, False), (1, 1937, 16, False),  # ViT-L/16 at 480^2, 736^2, 704^2
                 (2, 226, 12, False),                                              # ViT-B/32 at 480^2
                 (2, 25, 16, False), (2, 7, 12, False),                            # the test models
                 (2, 77, 12, True)]                                                # RN50x16's text tower width
# MHSA_SHAPES: the shapes tests/test_ops_gpu.py::test_mhsa runs every variant on (each there at amp 1 or 3)
SHAPES = [s[:4] for s in MHSA_SHAPES] + EDGE_SHAPES + ENGINE_SHAPES
FAMILIES = ["flat", "planted", "rising", "falling", "wide", "random1", "random3"]
VARIANTS = [None, 0, 3, 4]  # the engine's kernel, and one of each instantiation (lseg_mhsa_variant)


def _planted_pairs(N, causal):
    """{query row: dominant key}, at most one key per row, each pair on its own q / k channel."""
    keys = sorted({0, 63, 64, 127, 128, N - 1} & set(range(N)))
    rows = sorted({0, 1, 8, 63, 64, 65, 127, 128, 129, N // 2, N - 2, N - 1} & set(range(N)))
    pairs = {}
    if causal:
        for t in sorted((set(keys) | {1, 65, 129, 191, 192, N // 2}) & set(range(N))):
            pairs[t] = t  # the diagonal
        for r in rows:
            pairs.setdefault(r, max(k for k in keys if k <= r))
    else:
        for i, r in enumerate(rows):
            pairs[r] = keys[i % len(keys)]
    assert len(pairs) <= 64
    return pairs


def _qkv(family, B, N, heads, causal):
    D = heads * 64
    if family.startswith("random"):
        amp = 1.0 if family == "random1" else 3.0
        g = torch.Generator(device="cpu").manual_seed(19)
        return (torch.randn((B, N, 3 * D), generator=g) * amp).half().cuda()
    g = torch.Generator(device="cuda").manual_seed(1000 + FAMILIES.index(family))
    x = torch.randn((B, N, 3, heads, 64), generator=g, device="cuda")
    q, k, v = x[:, :, 0], x[:, :, 1], x[:, :, 2]
    t = torch.arange(N, device="cuda", dtype=torch.float32).view(1, N, 1)
    if family == "flat":
        q.zero_()
        v.copy_(torch.randint(-4, 5, v.shape, generator=g, device="cuda"))
    elif family == "planted":
        q.mul_(0.5)
        k.mul_(0.5)
        pairs = _planted_pairs(N, causal)
        for c, r in enumerate(pairs):
            q[:, r] = 0
            q[:, r, :, c] = 10.0  # score 100 * 0.125 = 12.5 nats, every other key of the row scores 0
            k[:, :, :, c] = 0
        for c, (r, key) in enumerate(pairs.items()):
            k[:, key, :, c] = 10.0
    elif family in ("rising", "falling"):
        q.mul_(0.5)
        k.mul_(0.5)
        q[..., 0] = 1.0
        k[..., 0] = (0.25 if family == "rising" else -0.25) * t  # 2 nats per 64-key tile
    elif family == "wide":
        q[..., 0] = 24.0
        k[..., 0] = 8.0 * (((37 * t) % 7) - 3)  # S spans +-576 on channel 0: ~210 log2 units
    return x.half().reshape(B, N, 3 * D).contiguous()


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("B,N,heads,causal", SHAPES)
def test_mhsa_families(ops, B, N, heads, causal, family):
    D = heads * 64
    qkv = _qkv(family, B, N, heads, causal)
    qkv_before = qkv.clone()
    ref, bound = mhsa_oracle(qkv, B, N, heads, causal)
    if family == "planted":  # the construction itself: each planted row's reference is its key's v row
        v = qkv.view(B, N, 3, heads, 64)[:, :, 2].double().reshape(B, N, D)
        for r, key in _planted_pairs(N, causal).items():
            assert torch.allclose(ref.view(B, N, D)[:, r], v[:, key], atol=0.05, rtol=0.05), (r, key)
    flat = flat_reference(qkv.view(B, N, 3, heads, 64)[:, :, 2], causal) if family == "flat" else None
    what = f"mhsa B={B} N={N} heads={heads} causal={causal} {family}"
    first = None
    for variant in VARIANTS:
        buf, out = _guarded(B * N, D)
        ops.mhsa(qkv, B, N, heads, causal, variant=variant, out=out)
        w = f"{what} variant {variant}"
        _guards_intact(buf, B * N, D, w)
        assert not torch.isnan(out).any(), f"{w}: NaN in the output (unwritten rows?)"
        n, msg = violations(out, ref, bound)
        assert n == 0, f"{w}: {msg}"
        if flat is not None:
            n, msg = violations(out, flat, flat_tolerance(flat, _eps_exp(variant)))
            assert n == 0, f"{w} (exact key count): {msg}"
        if variant is None:
            first = out.clone()
    # the same bits again, and each image alone equals its rows of the batch
    buf, again = _guarded(B * N, D)
    ops.mhsa(qkv, B, N, heads, causal, out=again)
    _same_bits(again, first, f"{what}: second run")
    if B > 1:
        for b in range(B):
            bb, one = _guarded(N, D)
            ops.mhsa(qkv[b], 1, N, heads, causal, out=one)
            _guards_intact(bb, N, D, f"{what} image {b} alone")
            _same_bits(one, first[b * N:(b + 1) * N], f"{what}: image {b} alone vs batched")
    _same_bits(qkv, qkv_before, f"{what}: qkv after the call")


def test_variant_instantiations(ops):
    """Variants 0, 1, 2, 5, 6 run one instantiation, 3 and 7 another, 4 and 8 a third: identical bits within each group;
    variant None is the one LSEG_MHSA_VARIANT names (default 0); lseg_mhsa_trace computes what variant 0 does."""
    B, N, heads = 2, 300, 3
    D = heads * 64
    for causal in (False, True):
        qkv = _qkv("random3", B, N, heads, causal)
        outs = {}
        for v in [None] + list(range(9)):
            buf, outs[v] = _guarded(B * N, D)
            ops.mhsa(qkv, B, N, heads, causal, variant=v, out=outs[v])
            _guards_intact(buf, B * N, D, f"variant {v}")
        for group in ([0, 1, 2, 5, 6], [3, 7], [4, 8]):
            for v in group[1:]:
                _same_bits(outs[v], outs[group[0]], f"causal={causal}: variant {v} vs {group[0]}")
        _same_bits(outs[None], outs[_env_variant()], f"causal={causal}: variant None vs {_env_variant()}")
        buf, tout = _guarded(B * N, D)
        _, trace = ops.mhsa_trace(qkv, B, N, heads, causal, out=tout)
        _guards_intact(buf, B * N, D, "mhsa_trace")
        _same_bits(tout, outs[0], f"causal={causal}: lseg_mhsa_trace vs variant 0")
        assert bool((trace != 0).any()), "mhsa_trace stamped nothing"


@pytest.mark.parametrize("side_stream", [False, True])
def test_pdl_chain(ops, side_stream):
    """QKV GEMM -> mhsa -> proj GEMM on one stream with no synchronisation in between (the kernels chain through
    programmatic dependent launch, as in every ViT block) must give the bits of the same three calls synchronised."""
    B, N, heads = 2, 901, 16
    D, M = heads * 64, B * N
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn((M, D), generator=g, device="cuda").half()
    wqkv = (torch.randn((3 * D, D), generator=g, device="cuda") * 0.06).half()
    bqkv = torch.randn((3 * D,), generator=g, device="cuda") * 0.1
    wproj = (torch.randn((D, D), generator=g, device="cuda") * 0.03).half()
    bproj = torch.randn((D,), generator=g, device="cuda") * 0.1

    def chain(sync, stream):
        qkv = torch.empty((M, 3 * D), dtype=torch.float16, device="cuda")
        buf, attn = _guarded(M, D)
        y = torch.empty((M, D), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            ops.gemm(x, wqkv, 3 * D, bias=bqkv, out_f16=qkv, ldc=3 * D)  # the engine's QKV GEMM: ldc = 3D
            if sync:
                torch.cuda.synchronize()
            ops.mhsa(qkv.view(B, N, 3 * D), B, N, heads, out=attn)
            if sync:
                torch.cuda.synchronize()
            ops.gemm(attn, wproj, D, bias=bproj, out_f32=y)
        torch.cuda.synchronize()
        _guards_intact(buf, M, D, f"chain sync={sync}")
        return qkv, attn, y

    want = chain(True, torch.cuda.current_stream())
    ref, bound = mhsa_oracle(want[0].view(B, N, 3 * D), B, N, heads, False)
    n, msg = violations(want[1], ref, bound)
    assert n == 0, f"synchronised chain: {msg}"
    stream = torch.cuda.Stream() if side_stream else torch.cuda.current_stream()
    got = chain(False, stream)
    for name, a, b in zip(("qkv", "attn", "proj"), got, want):
        bits = torch.int16 if a.dtype == torch.float16 else torch.int32
        assert torch.equal(a.view(bits), b.view(bits)), f"{name} differs between the PDL chain and the synchronised calls"


# ---------------------------------------------------------------------------------------------------------------------
# lseg_text_attn
# ---------------------------------------------------------------------------------------------------------------------
TEXT_SHAPES = [(1, 1, 8), (3, 2, 12), (3, 31, 8), (1, 32, 12), (3, 33, 8), (150, 63, 12), (3, 64, 8), (1, 65, 12),
               (23, 77, 8), (150, 77, 12), (512, 77, 8), (3, 80, 12), (512, 80, 12)]
TEXT_EXACT_MIN = 0.999  # bit-identical fraction against the emulation; measured on the H100: 1.0 at every shape


def _text_qkv(K, L, heads, seed):
    if (K, L, heads) == (23, 77, 8):  # the case this project tested before
        g = torch.Generator(device="cpu").manual_seed(31)
        return (torch.randn((K, L, 3 * heads * 64), generator=g) * 1.5).half().cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn((K, L, 3 * heads * 64), generator=g, device="cuda") * 1.5).half()


def _text_run(ops, qkv, K, L, heads, what):
    D = heads * 64
    buf, out = _guarded(K * L, D)
    ops.text_attn(qkv, K, L, heads, out=out)
    _guards_intact(buf, K * L, D, what)
    assert not torch.isnan(out).any(), f"{what}: NaN in the output (unwritten rows?)"
    return out


@pytest.mark.parametrize("K,L,heads", TEXT_SHAPES)
def test_text_attn_emulation(ops, K, L, heads):
    """lseg_text_attn follows torch's multi_head_attention_forward on fp16 tensors step by step (q scaled in fp16, bmm ->
    fp16, softmax -> fp16 normalised, bmm -> fp16), in the kernel's own summation order."""
    D = heads * 64
    what = f"text_attn K={K} L={L} heads={heads}"
    qkv = _text_qkv(K, L, heads, 40 + L)
    qkv_before = qkv.clone()
    got = _text_run(ops, qkv, K, L, heads, what)
    emu = text_attn_emulate(qkv, K, L, heads)
    diff = (got.double() - emu.double()).abs()
    far = diff > ulp16(emu.double())
    assert not far.any(), f"{what}: {int(far.sum())} elements more than 1 fp16 ulp from the emulation"
    exact = (got.view(torch.int16) == emu.view(torch.int16)).double().mean().item()
    assert exact >= TEXT_EXACT_MIN, f"{what}: only {exact:.5f} of the outputs bit-identical to the emulation"
    _same_bits(qkv, qkv_before, f"{what}: qkv after the call")
    # each label is independent: one label alone gives its rows of the batch
    for k in sorted({0, K // 2, K - 1}):
        one = _text_run(ops, qkv[k:k + 1].contiguous(), 1, L, heads, f"{what} label {k} alone")
        _same_bits(one, got[k * L:(k + 1) * L], f"{what}: label {k} alone vs batched")
    # q = 0: P_ij = fp16(1 / (i + 1)) and the PV chain are exactly emulable, so every bit must match
    flat = qkv.clone().view(K, L, 3, heads, 64)
    flat[:, :, 0] = 0
    flat = flat.view(K, L, 3 * D)
    got_flat = _text_run(ops, flat, K, L, heads, what + " flat")
    _same_bits(got_flat, text_attn_flat(flat.view(K, L, 3, heads, 64)[:, :, 2], K, L, heads), f"{what} flat")
    # the flash kernel on the same input (different rounding points, same function): within its float64 bound, and
    # close to the fp16-step recipe
    bm, mh = _guarded(K * L, D)
    ops.mhsa(qkv, K, L, heads, True, out=mh)
    _guards_intact(bm, K * L, D, what + " mhsa")
    ref, bound = mhsa_oracle(qkv, K, L, heads, True)
    n, msg = violations(mh, ref, bound)
    assert n == 0, f"{what}: mhsa(causal) {msg}"
    recipe = emu.double()
    err = (mh.double() - recipe).abs().max().item() / (recipe.abs().max().item() + 1e-12)
    assert err <= 3e-3, f"{what}: mhsa vs fp16-step recipe: max rel err {err:.3e}"


# ---------------------------------------------------------------------------------------------------------------------
# rejected arguments: an error naming the argument, nothing launched
# ---------------------------------------------------------------------------------------------------------------------
def _ptr(t, offset_bytes=0):
    import ctypes
    return None if t is None else ctypes.c_void_p(t.data_ptr() + offset_bytes)


def _stream():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rejected(call, match, bufs):
    from lseg_b200._lib import LsegError, check
    before = [b.clone() for b in bufs]
    with pytest.raises(LsegError, match=match):
        check(call())
    torch.cuda.synchronize()
    for b0, b1 in zip(before, bufs):
        _same_bits(b1, b0, f"rejected call ({match})")


def test_mhsa_rejects(ops):
    from lseg_b200._lib import load
    lib = load()
    B, N, heads = 2, 130, 2
    D = heads * 64
    big = torch.randn((B * N * 3 * D + 64,), device="cuda").half()
    qkv = big[:B * N * 3 * D]
    buf, out = _guarded(B * N, D)
    po = _ptr(out)

    def mhsa(q, o, b=B, n=N, h=heads):
        return lambda: lib.lseg_mhsa(q, o, b, n, h, 0, _stream())

    for b, n, h, name in [(0, N, heads, "B"), (-1, N, heads, "B"), (B, 0, heads, "N"), (B, -5, heads, "N"),
                          (B, N, 0, "heads"), (B, N, -2, "heads")]:
        _rejected(mhsa(_ptr(qkv), po, b, n, h), f"{name}=-?[0-9]+ must be positive", [buf])
    # B * heads > 65535 (gridDim.y); buffers big enough for the call, so a missing check could not fault
    Bx, hx = 4097, 16
    qx = torch.zeros((Bx * 3 * hx * 64,), dtype=torch.float16, device="cuda")
    bx, ox = _guarded(Bx, hx * 64)
    _rejected(lambda: lib.lseg_mhsa(_ptr(qx), _ptr(ox), Bx, 1, hx, 0, _stream()), "B\\*heads", [bx])
    _rejected(mhsa(None, po), "qkv pointer .* null", [buf])
    _rejected(mhsa(_ptr(qkv), None), "out pointer .* null", [buf])
    _rejected(mhsa(_ptr(big, 8), po), "qkv pointer .* not 16-byte aligned", [buf])
    _rejected(mhsa(_ptr(qkv), _ptr(out, 2)), "out pointer .* not 4-byte aligned", [buf])
    for v in (-1, 9):
        _rejected(lambda: lib.lseg_mhsa_variant(_ptr(qkv), po, B, N, heads, 0, v, _stream()), "variant", [buf])
    _rejected(lambda: lib.lseg_mhsa_trace(_ptr(qkv), po, B, N, heads, 0, None, _stream()), "trace", [buf])
    _rejected(lambda: lib.lseg_mhsa_trace(_ptr(qkv), _ptr(out, 2), B, N, heads, 0, _ptr(qx), _stream()),
              "out pointer", [buf])
    # the Python wrapper checks a caller-given out
    from lseg_b200._lib import LsegError
    for bad in (torch.zeros((B * N, D), dtype=torch.float32, device="cuda"),
                torch.zeros((B * N, D + 64), dtype=torch.float16, device="cuda")):
        before = bad.clone()
        with pytest.raises(LsegError, match="out must be fp16"):
            ops.mhsa(qkv.view(B, N, 3 * D), B, N, heads, out=bad)
        assert torch.equal(bad, before)


def test_text_attn_rejects(ops):
    from lseg_b200._lib import load
    lib = load()
    K, L, heads = 3, 77, 8
    D = heads * 64
    big = torch.randn((K * L * 3 * D + 64,), device="cuda").half()
    qkv = big[:K * L * 3 * D]
    buf, out = _guarded(K * L, D)

    def ta(q, o, k=K, l=L, h=heads):
        return lambda: lib.lseg_text_attn(q, o, k, l, h, _stream())

    for k, l, h, match in [(K, 0, heads, "L=0"), (K, 81, heads, "L=81"), (0, L, heads, "K=0"),
                           (65536, L, heads, "K=65536"), (K, L, 0, "heads=0"), (K, L, -1, "heads=-1")]:
        _rejected(ta(_ptr(qkv), _ptr(out), k, l, h), match, [buf])
    _rejected(ta(None, _ptr(out)), "qkv pointer", [buf])
    _rejected(ta(_ptr(qkv), None), "out pointer", [buf])
    _rejected(ta(_ptr(big, 2), _ptr(out)), "qkv pointer .* not 4-byte aligned", [buf])
    _rejected(ta(_ptr(qkv), _ptr(out, 2)), "out pointer .* not 4-byte aligned", [buf])
