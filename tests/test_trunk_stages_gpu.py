"""Every op of a traced image-trunk block, element by element, fed the engine's own input of that op.

lseg_debug_set_trace_block(j) makes the image plan snapshot block j's intermediates (trace_* debug buffers; the ViT's
patch_out and ResNet-101's stem / pool are always named). One forward per (case, traced block); then, per image, each
op of tests/trunk_oracle.py is checked against its float64 reference fed the engine's buffer that feeds it: tier A
(every element within the derived bound) and tier B (fp16 outputs mostly bit-identical to the rounded reference, fp32
outputs free of hidden fp16 roundings). Exact contracts on top, bit for bit:
  - ViT: a hooked block's trace_out is its tap, the next block's trace_in is that tap, block 0's trace_in is
    assemble_tokens(patch_out, cls, pos);
  - ResNet-101: trace_out16 = rn16(trace_out32), a stage's last block gives layer{L}, a stage's first block reads the
    previous stage's output (the pool output for stage 1), pool = maxpool(stem);
  - the logits and the launch count with the trace on equal those of the plan built with the trace off.
Each case prints one TRUNK json line: per op the worst err / bound ratio and the tier-B figure (worst block and image),
and the kernel instantiation, grid, split and cluster size of each trunk GEMM at the case's shapes.

LSEG_SPLITK and LSEG_SPLITK_FIXED are read once per process: a subprocess runs one case under each.
"""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import attention_oracle as A
import stage_oracle as S
import trunk_oracle as T
from parity_util import synth
from test_image_stages_gpu import _engine, _text

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F16, F32 = torch.float16, torch.float32
VITL, VITB, RN = "clip_vitl16_384", "clip_vitb32_384", "clip_resnet101"
K = 3


def _ops():
    import lseg_b200  # noqa: F401
    from lseg_b200 import ops
    return ops


def _eps_exp():
    """The exponential of the MHSA instantiation the engine runs (LSEG_MHSA_VARIANT, default 0: MUFU ex2)."""
    return A.EPS_POLY if int(os.environ.get("LSEG_MHSA_VARIANT", "0")) in (3, 4, 7, 8) else A.EPS_EX2


def _bits_equal(a, b):
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    iv = torch.int16 if a.element_size() == 2 else torch.int32
    return torch.equal(a.contiguous().view(iv), b.contiguous().view(iv))


class Report:
    def __init__(self):
        self.ops, self.fails = {}, []

    def add(self, rep, fails, f16s, where):
        for op, r in rep.items():
            old = self.ops.get(op)
            if old:
                r = {"worst": max(old["worst"], r["worst"]),
                     "tier_b": min(old["tier_b"], r["tier_b"]) if f16s[op] else max(old["tier_b"], r["tier_b"])}
            self.ops[op] = r
        self.fails += [f"{where} {f}" for f in fails]

    def check(self, ops, where):
        rep, fails = T.judge(ops)
        self.add(rep, fails, {k: v[2] for k, v in ops.items()}, where)

    def exact(self, name, ok):
        if not ok:
            self.fails.append(f"{name}: not bit-identical")


def _wt(n, k):
    return torch.empty((-(-n // 128) * 128, k), dtype=F16, device="cuda")


def _plan(ops, a, w, n, **kw):
    p, c = ops.gemm_plan(a, w, n, **kw), ops.gemm_cluster(a, w, n, **kw)
    return {"kernel": p["kernel"], "grid": p["grid"], "split_k": p["split_k"], "split_fixed": p["split_fixed"],
            "cluster": c["cluster"]}


# ------------------------------------------------------------------------------------------------------------------
# ViT
# ------------------------------------------------------------------------------------------------------------------
def _vit_gemms(ops, M, BT, D, P):
    """Plans of the trunk's GEMMs at this shape, planned the way build_vit_trunk plans them."""
    e = lambda *s, dt=F16: torch.empty(s, dtype=dt, device="cuda")  # noqa: E731
    x, b = e(M, D, dt=F32), e(4 * D, dt=F32)
    return {"patch": _plan(ops, e(BT, 3 * P * P), _wt(D, 3 * P * P), D, bias=b[:D], out_f32=e(BT, D, dt=F32)),
            "qkv": _plan(ops, e(M, D), _wt(3 * D, D), 3 * D, bias=b[:3 * D], out_f16=e(M, 3 * D)),
            "proj": _plan(ops, e(M, D), _wt(D, D), D, bias=b[:D], res_f32=x, out_f32=x),
            "fc1": _plan(ops, e(M, D), _wt(4 * D, D), 4 * D, bias=b, act=ops.ACT_GELU, out_f16=e(M, 4 * D)),
            "fc2": _plan(ops, e(M, 4 * D), _wt(D, 4 * D), D, bias=b[:D], res_f32=x, out_f32=x)}


def _segments(plan, M, N, Kd):
    return T.stream_k_segments(M, N, Kd, plan["grid"]) if plan["split_k"] else 1


def run_vit(bb, B, H, W, blocks, *, exact=True, expect_split=False, wrong_weights_block=None, name=None):
    from lseg_b200.packing import BACKBONES
    ops = _ops()
    cfg = BACKBONES[bb]
    D, P, heads, depth, hooks = cfg["dim"], cfg["patch"], cfg["heads"], cfg["depth"], cfg["hooks"]
    gh, gw = H // P, W // P
    Tn = gh * gw
    N, M = Tn + 1, B * (Tn + 1)
    eng, sd = _engine(bb)
    x = synth.make_image(B, H, W, seed=B * 1000 + H + W).cuda()
    text = _text(eng.padded_rows(K), eng.out_c, H + W).cuda()
    ops.set_trace_block(-1)
    rep = Report()
    try:
        logits = eng.forward(x, text, K).clone()
        launches = eng.last_launch_count()
        taps = [eng.debug_tensor(f"tap{k}", (M, D), F32).clone() for k in range(4)]
        gemms = _vit_gemms(ops, M, B * Tn, D, P)
        if expect_split:
            assert gemms["fc2"]["split_k"] == 1, gemms
        seg_proj, seg_fc2 = _segments(gemms["proj"], M, D, D), _segments(gemms["fc2"], M, D, 4 * D)
        pw, pb = sd["pretrained.model.patch_embed.proj.weight"].cuda(), sd["pretrained.model.patch_embed.proj.bias"]
        for j in blocks:
            ops.set_trace_block(j)
            out = eng.forward(x, text, K)
            torch.cuda.synchronize()
            assert eng.last_launch_count() == launches, (j, eng.last_launch_count(), launches)
            if exact:
                rep.exact(f"block {j}: logits with the trace on", _bits_equal(out, logits))
            shapes = {"trace_in": (D, F32), "trace_ln1": (D, F16), "trace_qkv": (3 * D, F16), "trace_attn": (D, F16),
                      "trace_x1": (D, F32), "trace_ln2": (D, F16), "trace_fc1": (4 * D, F16), "trace_out": (D, F32)}
            tr = {n: eng.debug_tensor(n, (M, c), dt) for n, (c, dt) in shapes.items()}
            patch_out = eng.debug_tensor("patch_out", (B * Tn, D), F32)
            if j == blocks[0]:
                for b in range(B):
                    rep.check({"patch": (patch_out[b * Tn:(b + 1) * Tn], T.patch_embed(x[b:b + 1], pw, pb), False)},
                              f"image {b}")
            if j == 0:
                pos = ops.pos_resize(sd["pretrained.model.pos_embed"].reshape(-1, D).float().cuda().contiguous(),
                                     int(round(((sd["pretrained.model.pos_embed"].shape[1] - 1) ** 0.5))), gh, gw)
                cls = sd["pretrained.model.cls_token"].reshape(D).float().cuda()
                rep.exact("block 0: trace_in = assemble_tokens(patch_out, cls, pos)",
                          _bits_equal(tr["trace_in"], ops.assemble_tokens(patch_out, cls, pos, B, Tn).reshape(M, D)))
            for k, hk in enumerate(hooks):
                if j == hk:
                    rep.exact(f"block {j}: trace_out = tap{k}", _bits_equal(tr["trace_out"], taps[k]))
                if j == hk + 1:
                    rep.exact(f"block {j}: trace_in = tap{k}", _bits_equal(tr["trace_in"], taps[k]))
            p = T.vit_block_params(sd, j, "cuda")
            for b in range(B):
                one = {n: t[b * N:(b + 1) * N] for n, t in tr.items()}
                rep.check(T.vit_block(one, p, heads, eps_exp=_eps_exp(), seg_proj=seg_proj, seg_fc2=seg_fc2),
                          f"block {j} image {b}")
                if j == wrong_weights_block:  # non-vacuity: block j + 1's weights are far outside every bound
                    wrong, _ = T.judge(T.vit_block(one, T.vit_block_params(sd, j + 1, "cuda"), heads,
                                                   eps_exp=_eps_exp(), seg_proj=seg_proj, seg_fc2=seg_fc2))
                    passed = [op for op, r in wrong.items() if op != "mhsa" and r["worst"] <= 1.0]
                    assert not passed, f"block {j + 1}'s weights pass tier A on block {j}'s trace: {passed}"
    finally:
        ops.set_trace_block(-1)
    print("TRUNK " + json.dumps({"case": name or f"{bb}_B{B}_{H}x{W}_blocks{list(blocks)}", "ops": rep.ops,
                                 "gemms": gemms, "segments": {"proj": seg_proj, "fc2": seg_fc2}}))
    assert not rep.fails, rep.fails[:20]


# ------------------------------------------------------------------------------------------------------------------
# ResNet-101
# ------------------------------------------------------------------------------------------------------------------
LAYERS = (3, 4, 23, 3)


def _rn_block_geometry(blk, B, H, W):
    """(stage, index in stage, stride, input (h, w), output (h, w), cin, width, cout) of global bottleneck blk."""
    L, i = 0, blk
    while i >= LAYERS[L]:
        i -= LAYERS[L]
        L += 1
    h0, w0 = H // 4, W // 4
    stride = 2 if (L > 0 and i == 0) else 1
    ho, wo = h0 >> L, w0 >> L
    hi, wi = (ho * stride, wo * stride)
    width = 64 << L
    cout = 4 * width
    cin = cout if i > 0 else (64 if L == 0 else 2 * width)
    return L, i, stride, (hi, wi), (ho, wo), cin, width, cout


def _rn_gemms(ops, B, hi, wi, ho, wo, stride, cin, width, cout, t1):
    e = lambda *s, dt=F16: torch.empty(s, dtype=dt, device="cuda")  # noqa: E731
    pxi, px = B * hi * wi, B * ho * wo
    s, y = e(cout, dt=F32), e(px, cout, dt=F32)
    g = {"conv1": _plan(ops, e(pxi, cin), _wt(width, cin), width, scale=s[:width], bias=s[:width], act=ops.ACT_RELU,
                        out_f16=e(pxi, width))}
    if stride == 1:
        g["conv2"] = _plan(ops, t1, _wt(width, 9 * width), width, conv=(3, 1), scale=s[:width], bias=s[:width],
                           act=ops.ACT_RELU, out_f16=e(px, width))
    else:
        g["conv2"] = _plan(ops, e(px, 9 * width), _wt(width, 9 * width), width, scale=s[:width], bias=s[:width],
                           act=ops.ACT_RELU, out_f16=e(px, width))
    g["conv3"] = _plan(ops, e(px, width), _wt(cout, width), cout, scale=s, bias=s, res_f32=y, out_f32=y,
                       out_f16=e(px, cout), relu_after_res=True)
    return g


def run_rn(B, H, W, blocks, *, exact=True, expect_fixed_split=0, wrong_weights_block=None, name=None):
    ops = _ops()
    eng, sd = _engine(RN)
    x = synth.make_image(B, H, W, seed=B * 1000 + H + W).cuda()
    text = _text(eng.padded_rows(K), eng.out_c, H + W).cuda()
    ops.set_trace_block(-1)
    rep, gemms = Report(), {}
    sizes = [(H // 4 >> L, W // 4 >> L, 256 << L) for L in range(4)]
    try:
        logits = eng.forward(x, text, K).clone()
        launches = eng.last_launch_count()
        layers = [eng.debug_tensor(f"layer{L}", (B, h, w, c), F16).clone() for L, (h, w, c) in enumerate(sizes)]
        for n, j in enumerate(blocks):
            L, i, stride, (hi, wi), (ho, wo), cin, width, cout = _rn_block_geometry(j, B, H, W)
            ops.set_trace_block(j)
            out = eng.forward(x, text, K)
            torch.cuda.synchronize()
            assert eng.last_launch_count() == launches, (j, eng.last_launch_count(), launches)
            if exact:
                rep.exact(f"block {j}: logits with the trace on", _bits_equal(out, logits))
            get = eng.debug_tensor
            tr = {"trace_in": get("trace_in", (B, hi, wi, cin), F16), "trace_t1": get("trace_t1", (B, hi, wi, width), F16),
                  "trace_t2": get("trace_t2", (B, ho, wo, width), F16),
                  "trace_id": get("trace_id", (B, ho, wo, cout), F32),
                  "trace_out32": get("trace_out32", (B, ho, wo, cout), F32),
                  "trace_out16": get("trace_out16", (B, ho, wo, cout), F16)}
            stem = get("stem", (B, H // 2, W // 2, 64), F16)
            pool = get("pool", (B, H // 4, W // 4, 64), F16)
            if n == 0:
                st_w = sd["pretrained.layer1.0.weight"].cuda()
                bn = tuple(t.cuda() for t in S.fold_bn(sd, "pretrained.layer1.1."))
                for b in range(B):
                    rep.check({"stem": (stem[b:b + 1], T.stem(x[b:b + 1], st_w, bn), True)}, f"image {b}")
                mp = F.max_pool2d(stem.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
                rep.exact("pool = maxpool(stem)", _bits_equal(pool, mp.contiguous()))
            rep.exact(f"block {j}: trace_out16 = rn16(trace_out32)", _bits_equal(tr["trace_out16"], tr["trace_out32"].half()))
            if i == LAYERS[L] - 1:
                rep.exact(f"block {j}: trace_out16 = layer{L}", _bits_equal(tr["trace_out16"], layers[L]))
            if i == 0:
                prev = pool if L == 0 else layers[L - 1]
                rep.exact(f"block {j}: trace_in = the previous stage's output", _bits_equal(tr["trace_in"], prev))
            for k, v in _rn_gemms(ops, B, hi, wi, ho, wo, stride, cin, width, cout, tr["trace_t1"]).items():
                gemms[f"{k}_stage{L + 1}_s{stride}"] = v
            p, st = T.bottleneck_params(sd, j, LAYERS, "cuda")
            assert st == stride
            for b in range(B):
                one = {nm: t[b:b + 1] for nm, t in tr.items()}
                rep.check(T.bottleneck(one, p, stride), f"block {j} image {b}")
                if j == wrong_weights_block:  # non-vacuity: block j + 1's weights (same stage, same shapes)
                    wrong, _ = T.judge(T.bottleneck(one, T.bottleneck_params(sd, j + 1, LAYERS, "cuda")[0], stride))
                    passed = [op for op, r in wrong.items() if r["worst"] <= 1.0]
                    assert not passed, f"block {j + 1}'s weights pass tier A on block {j}'s trace: {passed}"
        if expect_fixed_split:
            assert any(g["split_fixed"] == expect_fixed_split for g in gemms.values()), gemms
    finally:
        ops.set_trace_block(-1)
    print("TRUNK " + json.dumps({"case": name or f"{RN}_B{B}_{H}x{W}_blocks{list(blocks)}", "ops": rep.ops,
                                 "gemms": gemms}))
    assert not rep.fails, rep.fails[:20]


# ------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------
# B=1 32x32: N = 5, one partial M tile; 160x224: a non-square pos-embed resize; 480^2: M = 1802 and, at B = 8, the 2-CTA
# paired GEMMs; 704^2: N = 1937 (BASELINE.json configs[4])
@pytest.mark.parametrize("B,H,W,blocks", [(1, 32, 32, (0, 23)), (2, 64, 96, (0, 6, 23)), (2, 160, 224, (11,)),
                                          (2, 480, 480, (0, 5, 6, 12, 23)), (8, 480, 480, (23,)),
                                          (1, 704, 704, (12,))])
def test_trunk_vitl16(B, H, W, blocks):
    run_vit(VITL, B, H, W, blocks, wrong_weights_block=6 if (B, H, W) == (2, 64, 96) else None)


def test_trace_block_rejects():
    """Below -1: rejected by the setter, nothing changes. At or past the block count: the next forward fails, naming the
    trace block and the block count, and leaves its output untouched."""
    from lseg_b200._lib import LsegError
    ops = _ops()
    eng, _ = _engine(VITL)
    B, H, W = 1, 32, 32
    x = synth.make_image(B, H, W, seed=5).cuda()
    text = _text(eng.padded_rows(K), eng.out_c, 5).cuda()
    ops.set_trace_block(-1)
    logits = eng.forward(x, text, K).clone()
    launches = eng.last_launch_count()
    try:
        with pytest.raises(LsegError, match=r"debug_set_trace_block: .*got -2"):
            ops.set_trace_block(-2)
        out = torch.full_like(logits, float("nan"))
        eng.forward(x, text, K, out=out)
        assert _bits_equal(out, logits) and eng.last_launch_count() == launches
        with pytest.raises(KeyError):  # the rejected value did not turn the trace on
            eng.debug_tensor("trace_in", (B * 5, 1024), F32)
        for bad in (24, 1000):
            ops.set_trace_block(bad)
            out = torch.full_like(logits, 7.0)
            with pytest.raises(LsegError, match=rf"trace block {bad} .* 24 blocks"):
                eng.forward(x, text, K, out=out)
            torch.cuda.synchronize()
            assert bool((out == 7.0).all()), "a rejected forward wrote its output"
        ops.set_trace_block(23)  # the last block is accepted
        eng.forward(x, text, K, out=out)
        assert _bits_equal(out, logits)
    finally:
        ops.set_trace_block(-1)


def test_trace_under_cluster_modes():
    """Unclustered (1) and clustered-wherever-possible (3) GEMM plans give the default plan's trace bits."""
    ops = _ops()
    eng, _ = _engine(VITL)
    B, H, W, j = 2, 64, 96, 6
    x = synth.make_image(B, H, W, seed=11).cuda()
    text = _text(eng.padded_rows(K), eng.out_c, 11).cuda()
    names = ["trace_in", "trace_ln1", "trace_qkv", "trace_attn", "trace_x1", "trace_ln2", "trace_fc1", "trace_out"]
    M, D = B * ((H // 16) * (W // 16) + 1), 1024
    width = {"trace_qkv": 3 * D, "trace_fc1": 4 * D}
    dtype = {"trace_in": F32, "trace_x1": F32, "trace_out": F32}

    def trace():
        eng.forward(x, text, K)
        torch.cuda.synchronize()
        return {n: eng.debug_tensor(n, (M, width.get(n, D)), dtype.get(n, F16)).clone() for n in names}

    try:
        ops.set_trace_block(j)
        want = trace()
        for mode in (1, 3):
            ops.set_gemm_cluster(mode)
            got = trace()
            bad = [n for n in names if not _bits_equal(got[n], want[n])]
            assert not bad, f"cluster mode {mode}: {bad} differ from the default plan's"
    finally:
        ops.set_gemm_cluster(2)
        ops.set_trace_block(-1)


@pytest.mark.parametrize("B,H,W,blocks", [(3, 160, 224, (0, 8, 11)), (2, 480, 480, (2, 3))])
def test_trunk_vitb32(B, H, W, blocks):
    run_vit(VITB, B, H, W, blocks)


# B=1 32x32: stage 4 at 1x1, so 8 of the 9 taps of its 3x3 convs are padding
@pytest.mark.parametrize("B,H,W,blocks", [(1, 32, 32, (0, 3, 30, 32)), (3, 96, 128, (0, 3, 4, 7, 29, 30, 32)),
                                          (2, 480, 480, (3, 7, 30))])
def test_trunk_resnet101(B, H, W, blocks):
    run_rn(B, H, W, blocks, wrong_weights_block=4 if (B, H, W) == (3, 96, 128) else None)


def test_trace_block_rejects_resnet():
    from lseg_b200._lib import LsegError
    ops = _ops()
    eng, _ = _engine(RN)
    x = synth.make_image(1, 32, 32, seed=6).cuda()
    text = _text(eng.padded_rows(K), eng.out_c, 6).cuda()
    out = torch.full((1, K, 32, 32), 7.0, device="cuda")
    ops.set_trace_block(33)
    try:
        with pytest.raises(LsegError, match=r"trace block 33 .* 33 blocks"):
            eng.forward(x, text, K, out=out)
        torch.cuda.synchronize()
        assert bool((out == 7.0).all()), "a rejected forward wrote its output"
    finally:
        ops.set_trace_block(-1)


_SWITCH_SCRIPT = """
import sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import lseg_b200
import test_trunk_stages_gpu as T
if sys.argv[2] == "vit":
    T.run_vit(T.VITL, 8, 480, 480, (23,), exact=False, expect_split=True, name="switch_LSEG_SPLITK=1")
else:
    T.run_rn(3, 96, 128, (0, 3, 4, 7, 29, 30, 32), expect_fixed_split=3, name="switch_LSEG_SPLITK_FIXED=3")
"""


@pytest.mark.parametrize("which,env", [("vit", {"LSEG_SPLITK": "1"}), ("rn", {"LSEG_SPLITK_FIXED": "3"})])
def test_trunk_under_switches(which, env):
    """LSEG_SPLITK=1: fc2 at B = 8, 480^2 takes the stream-K split (several reduce-adds per tile, in no fixed order, so
    the logits are compared by bound only). LSEG_SPLITK_FIXED=3: three-way split-K of the stride-1 3x3 convs. Every bound
    and tier holds unchanged."""
    r = subprocess.run([sys.executable, "-c", _SWITCH_SCRIPT, ROOT, which], env=dict(os.environ, **env),
                       capture_output=True, text=True, timeout=1800)
    print(r.stdout[-20000:])
    assert r.returncode == 0, r.stderr[-5000:]
