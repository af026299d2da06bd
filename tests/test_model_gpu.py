"""GPU parity of the whole forward path (through the drop-in LSegNet and the C ABI) against the CPU
oracle on the same seeded weights and inputs.

Tolerance policy (every case prints its measurements as one PARITY json line; metric = max|got - ref| / max|ref|, the
"1e-3 relative fp16 tolerance" of BASELINE.json's north_star):

  * fp32 quantities of the oracle — the four ViT taps and the decoder output path_1 — are held to the contract as
    written: 1e-3 (STAGE_TOL; measured <= 8.9e-4 on every case).
  * the LOGITS are an fp16 tensor in the reference (`logit_scale * image_features.half() @ text_features.t()`,
    lseg_net.py:194, then .float() and a bilinear blend), so two correct evaluations may differ by one fp16 quantum of the
    logit scale wherever an fp32 sum lands on the other side of a rounding boundary: with the seeded weights max|logit|
    is 1.1-1.7, i.e. ONE quantum (2^-10) is already 6-9e-4 of max|logit|. The bar is therefore
        |got - ref| <= 1e-3 * max|ref| + 1 fp16 quantum(max|ref|)          (logit_tolerance(ref, 1e-3))
    for the image path + head + pixel x text + upsample with TEACHER-FORCED text features (the oracle's own fp16 text
    features fed to lseg_forward); measured 1.1-1.5e-3 where max|logit| ~ 1.2-1.7 and 8.6e-4 on the planted-prototype
    case (max|logit| 6.8), where the quantum is relatively small.
  * the CLIP text tower is a 12-layer fp16 network; with the seeded random weights it amplifies 1-ulp differences of the
    fp32 summation order to ~1.7e-3 of the feature scale at its output. That is a property of the reference: its own two
    executions — torch's nn.MultiheadAttention fast path inside the unmodified reference modules (committed as
    tests/golden/ref_480_k150.npz) and the step-by-step multi_head_attention_forward recipe the oracle restates — differ
    by 1.75e-3 (features), 2.0e-3 (logits), agree on 98.1 % of the argmax pixels and flip pixels whose top-2 margin is up
    to 4.8 fp16 quanta (tests/test_oracle.py::test_480_golden_matches_oracle[k150], CPU; tools/text_tower_floor.py).
    So the tower is held to (a) op-level parity with teacher-forced inputs: every op of a block, fed the oracle's own
    input, reproduces the oracle's output to one fp16 ulp with >= 99 % of the elements bit-identical (each op follows the
    reference's rounding points); (b) block-level: <= 3 quanta of the residual-stream scale; (c) end to end: no further
    from the oracle — and from the reference's own golden features — than TEXT_FLOOR_FACTOR x the distance between the
    reference's two executions. Full-pipeline logits (own text tower): logit_tolerance(ref, FULL_LOGIT_REL).
  * argmax masks: identical, except pixels whose ORACLE top-2 margin is below a few fp16 quanta of the logit scale
    (ties that another summation order may break differently): MARGIN_QUANTA_TF = 3 with teacher-forced text (measured
    worst 1.5), MARGIN_QUANTA_FULL = 6 with the GPU text tower (measured worst 4.1; the reference's own two executions:
    4.8). Cases with real margins (K = 2, planted prototypes) must match exactly / to 1e-4.
"""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from parity_util import (NET_KW, argmax_report, argmax_report_from_mask, on_lattice, oracle_forward, oracle_threads, rel_err,
                         rms_rel_err, state_dict, synth)

pytestmark = pytest.mark.gpu
oracle_threads()

STAGE_TOL = 1.0e-3        # taps of blocks 5/11/17/23 and path_1, relative to max|ref|
LOGIT_REL = 1.0e-3        # logits, teacher-forced text features: + one fp16 quantum of the logit scale (logit_tolerance)
FULL_LOGIT_REL = 3.0e-3   # logits with the GPU text tower (reference-vs-reference floor: 2.0e-3), + one quantum
TEXT_FLOOR_FACTOR = 1.5   # GPU text features vs oracle <= 1.5 x (reference fast path vs oracle)
MARGIN_QUANTA_TF = 3
MARGIN_QUANTA_FULL = 6
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def fp16_quantum(v):
    return 2.0 ** (math.floor(math.log2(max(float(v), 2.0 ** -14))) - 10)


def logit_tolerance(ref, rel):
    """allowed max|got - ref| / max|ref| for an fp16-valued logits tensor: rel + one fp16 quantum of its scale"""
    mx = float(ref.abs().max())
    return rel + fp16_quantum(mx) / mx


def margin_eps(ref, quanta=MARGIN_QUANTA_FULL):
    return quanta * fp16_quantum(ref.abs().max())


@pytest.fixture(scope="module")
def net():
    import lseg_b200  # noqa: F401
    from lseg_b200.lseg_net import LSegNet
    labels = synth.ade20k_labels()
    n = LSegNet(labels=labels, **NET_KW)
    n.load_state_dict(state_dict(0))
    return n.cuda().eval()


def _report(name, d):
    print("PARITY " + json.dumps({"case": name, **d}))
    out = os.path.join(os.path.dirname(__file__), "..", "gpurun_out")
    if os.path.isdir(out):
        with open(os.path.join(out, "parity.jsonl"), "a") as f:
            f.write(json.dumps({"case": name, **d}) + "\n")


def _padded_text(eng, feats):
    """oracle fp16 text features [K,512] -> the engine's operand layout (rows padded to 128, zero rows)."""
    k = feats.shape[0]
    t = torch.zeros((eng.padded_rows(k), feats.shape[1]), dtype=torch.float16, device="cuda")
    t[:k] = feats.half().cuda()
    return t


# ------------------------------------------------------------------------------------------------
# CLIP text tower
# ------------------------------------------------------------------------------------------------
def test_text_encoder_end_to_end(net):
    from oracle import lseg_oracle as O
    tokens = synth.tokenize(synth.ade20k_labels())
    eng = net._engine_for(torch.device("cuda"))
    got = eng.encode_text(tokens)[:150].float().cpu()
    tw = O.clip_text_weights_fp16(state_dict(0))
    ref = O.clip_encode_text(tokens, tw).float()
    ref = ref / ref.norm(dim=-1, keepdim=True)
    gold = torch.from_numpy(np.load(os.path.join(GOLD, "ref_480_k150.npz"))["text_features"]).float()
    floor = rel_err(gold, ref)  # the reference's own two executions of this tower
    cos = F.cosine_similarity(got, ref, dim=-1)
    d = {"vs_oracle": rel_err(got, ref), "vs_reference_golden": rel_err(got, gold), "reference_vs_oracle_floor": floor,
         "rms_vs_oracle": rms_rel_err(got, ref), "min_cos": cos.min().item()}
    _report("text_encoder_k150", d)
    assert 1.0e-3 < floor < 2.5e-3, floor  # the fixture still shows the floor this policy rests on
    assert d["vs_oracle"] <= TEXT_FLOOR_FACTOR * floor, d
    assert d["vs_reference_golden"] <= TEXT_FLOOR_FACTOR * floor, d
    assert d["min_cos"] > 0.99999, d


def _ulp16(ref, floor):
    return torch.clamp(ref.abs(), min=floor).log2().floor().exp2() * 2.0 ** -10


def test_text_ops_teacher_forced():
    """Every op of a ResidualAttentionBlock, fed the ORACLE's own input of that op, against the oracle's output of that
    op (blocks 0, 5 and 11): LayerNorm, in_proj GEMM, lseg_text_attn, out_proj GEMM + fp16 residual, LayerNorm, c_fc GEMM +
    QuickGELU, c_proj GEMM + fp16 residual — all through the C ABI stage ops. Each op must be within ONE fp16 ulp of the
    oracle (two for the residual adds, whose ulp is taken at the operand scale) with >= 99 % of the elements
    bit-identical: the rounding points are the reference's, what remains is the order of fp32 sums. The whole block,
    chained on the GPU from the oracle's block input, must stay within 3 quanta of the residual-stream scale."""
    from lseg_b200 import ops
    from oracle import lseg_oracle as O
    sd = state_dict(0)
    tw = O.clip_text_weights_fp16(sd)
    tokens = synth.tokenize(synth.ade20k_labels()[:40])
    K, L, Wd = tokens.shape[0], 77, 512
    M = K * L
    io, tr = [], {0: {}, 5: {}, 11: {}}
    O.clip_encode_text(tokens, tw, layer_io=io, op_trace=tr)
    report = {}

    def dev(t, cols):  # oracle activation [K,77,cols] -> padded fp16 rows on the GPU (TMA boxes never exceed the tensor)
        return ops.pad_rows(t.reshape(M, cols).half().cuda())

    def check(name, got, ref, max_ulp):
        # error in fp16 ulps of the element, but never finer than the ulp at 1/8 of the tensor's largest magnitude: an
        # output that is small by cancellation (a dot product near zero) carries the rounding of its O(max) terms
        got, ref = got[:M].float().cpu(), ref.reshape(M, -1).float()
        diff = (got - ref).abs()
        worst = (diff / _ulp16(ref, float(ref.abs().max()) / 8)).max().item()
        exact = (diff == 0).float().mean().item()
        report[name] = (round(worst, 2), round(exact, 4))
        assert worst <= max_ulp, (name, worst, exact)
        assert exact >= 0.99, (name, worst, exact)

    for i, t in tr.items():
        b = f"transformer.resblocks.{i}."

        def wt(name):
            return ops.pad_rows(tw[b + name].half().cuda())

        def bias(name):
            return tw[b + name].float().cuda()

        x0 = dev(io[i], Wd)
        scale = float(io[i + 1].abs().max())
        # -- each op on the oracle's input of that op --
        h = ops.layernorm(x0, tw[b + "ln_1.weight"].cuda(), tw[b + "ln_1.bias"].cuda(), 1e-5)
        check(f"b{i}.ln1", h, t["ln1"], 1.0)
        qkv = torch.empty((x0.shape[0], 3 * Wd), dtype=torch.float16, device="cuda")
        ops.gemm(dev(t["ln1"], Wd), wt("attn.in_proj_weight"), 3 * Wd, M=M, bias=bias("attn.in_proj_bias"), out_f16=qkv)
        check(f"b{i}.in_proj", qkv, t["qkv"], 1.0)
        a = ops.text_attn(t["qkv"].half().cuda().contiguous(), K, L, 8)
        check(f"b{i}.attn", a, t["attn"], 1.0)
        x1 = torch.zeros_like(x0)
        ops.gemm(dev(t["attn"], Wd), wt("attn.out_proj.weight"), Wd, M=M, bias=bias("attn.out_proj.bias"), res_f16=x0,
                 out_f16=x1)
        check(f"b{i}.out_proj+res", x1, t["x1"], 2.0)
        h2 = ops.layernorm(dev(t["x1"], Wd), tw[b + "ln_2.weight"].cuda(), tw[b + "ln_2.bias"].cuda(), 1e-5)
        check(f"b{i}.ln2", h2, t["ln2"], 1.0)
        g = torch.empty((x0.shape[0], 4 * Wd), dtype=torch.float16, device="cuda")
        ops.gemm(dev(t["ln2"], Wd), wt("mlp.c_fc.weight"), 4 * Wd, M=M, bias=bias("mlp.c_fc.bias"), act=ops.ACT_QUICKGELU,
                 out_f16=g)
        # a 1-ulp flip of the pre-activation h (summation order) moves x*sigmoid(1.702x) by up to ~3 of ITS ulps where the
        # output is much smaller than h (negative h): allow 4
        check(f"b{i}.c_fc+quickgelu", g, t["gelu"], 4.0)
        x2 = torch.zeros_like(x0)
        ops.gemm(dev(t["gelu"], 4 * Wd), wt("mlp.c_proj.weight"), Wd, M=M, bias=bias("mlp.c_proj.bias"),
                 res_f16=dev(t["x1"], Wd), out_f16=x2)
        check(f"b{i}.c_proj+res", x2, t["x2"], 2.0)
        # -- the whole block chained on the GPU from the oracle's block input --
        ops.gemm(h, wt("attn.in_proj_weight"), 3 * Wd, M=M, bias=bias("attn.in_proj_bias"), out_f16=qkv)
        a = ops.pad_rows(ops.text_attn(qkv[:M].contiguous(), K, L, 8))
        ops.gemm(a, wt("attn.out_proj.weight"), Wd, M=M, bias=bias("attn.out_proj.bias"), res_f16=x0, out_f16=x1)
        h2 = ops.layernorm(x1, tw[b + "ln_2.weight"].cuda(), tw[b + "ln_2.bias"].cuda(), 1e-5)
        ops.gemm(h2, wt("mlp.c_fc.weight"), 4 * Wd, M=M, bias=bias("mlp.c_fc.bias"), act=ops.ACT_QUICKGELU, out_f16=g)
        ops.gemm(g, wt("mlp.c_proj.weight"), Wd, M=M, bias=bias("mlp.c_proj.bias"), res_f16=x1, out_f16=x2)
        blk = (x2[:M].float().cpu() - io[i + 1].reshape(M, Wd).float()).abs().max().item() / fp16_quantum(scale)
        report[f"b{i}.block_quanta"] = round(blk, 2)
        assert blk <= 3.0, (i, blk)
    _report("text_ops_teacher_forced", report)


# ------------------------------------------------------------------------------------------------
# image path
# ------------------------------------------------------------------------------------------------
# configs[1] (B=8 and B=1) / configs[0] of BASELINE.json plus small, non-square and odd-label-count shapes (partial M / N
# tiles, token grids that are not square, label counts that are not a multiple of 8)
@pytest.mark.parametrize("B,H,W,K", [(2, 64, 96, 5), (1, 480, 480, 150), (1, 480, 480, 2), (2, 160, 224, 7),
                                     (1, 320, 512, 33), (8, 480, 480, 150)])
def test_forward_vs_oracle(net, B, H, W, K):
    labels = synth.ade20k_labels()[:K] if K != 2 else ["cat", "other"]
    tokens = synth.tokenize(labels)
    x = synth.make_image(B, H, W, seed=B * 1000 + H)
    ref, st = oracle_forward(x, tokens)
    eng = net._engine_for(torch.device("cuda"))
    # (1) teacher-forced text features: everything but the text tower, at the contract's tolerance
    got_tf = eng.forward(x.cuda(), _padded_text(eng, st["text_features"]), K)
    N = (H // 16) * (W // 16) + 1
    d = {"launches": eng.last_launch_count()}
    for k in range(4):
        tap = eng.debug_tensor(f"tap{k}", (B, N, 1024), torch.float32)
        d[f"tap{k}"] = rel_err(tap, st["taps"][k])
    p1 = eng.debug_tensor("path1", (B, H // 2, W // 2, 256), torch.float16)
    d["path1"] = rel_err(p1.permute(0, 3, 1, 2), st["path_1"])
    d["logits_teacher_forced"] = rel_err(got_tf, ref)
    d["max_abs_logit"] = ref.abs().max().item()
    d["logit_tol_tf"] = logit_tolerance(ref, LOGIT_REL)
    d["logit_tol_full"] = logit_tolerance(ref, FULL_LOGIT_REL)
    tf = argmax_report(got_tf, ref, margin_eps(ref, MARGIN_QUANTA_TF))
    d.update({"tf_" + k: v for k, v in tf.items()})
    # (2) the public call: own text tower
    got = net(x.cuda(), tokens)
    assert got.shape == ref.shape and got.dtype == torch.float32 and got.is_contiguous()
    d["logits"] = rel_err(got, ref)
    d["logits_rms"] = rms_rel_err(got, ref)
    full = argmax_report(got, ref, margin_eps(ref))
    d.update(full)
    _report(f"forward_B{B}_{H}x{W}_K{K}", d)
    assert torch.isfinite(got).all() and torch.isfinite(got_tf).all()
    for k in range(4):
        assert d[f"tap{k}"] <= STAGE_TOL, d
    assert d["path1"] <= STAGE_TOL, d
    assert d["logits_teacher_forced"] <= d["logit_tol_tf"], d
    assert tf["ok"], d
    assert d["logits"] <= d["logit_tol_full"], d
    assert full["ok"], d
    if K == 2:  # configs[0]: real margins -> the mask is bit-identical
        assert tf["mismatch"] == 0 and full["mismatch"] == 0, d


# ------------------------------------------------------------------------------------------------
# the other backbones of lseg_net.py:119-123
#   clip_vitb32_384 (lseg_vit.py:259-405): ViT-B/32 trunk (D 768, 12 blocks, 12 heads, patch 32, hooks 2/5/8/11),
#     reassemble to 96/192/384/768 channels (stored 128/192/384/768) with ConvT x8 / x4 / x2 / none
#   clipRN50x16_vitl16_384 (lseg_vit.py:240-257): the ViT-L/16 trunk with CLIP RN50x16's text tower (width 768, 12 heads),
#     out_c = 768 (lseg_net.py:142-146)
# ------------------------------------------------------------------------------------------------
OTHER = {"b32": dict(backbone="clip_vitb32_384", D=768, patch=32, stored=(128, 192, 384, 768)),
         "rn50x16": dict(backbone="clipRN50x16_vitl16_384", D=1024, patch=16, stored=(256, 512, 1024, 1024))}
_OTHER_NETS = {}


def other_net(tag):
    if tag not in _OTHER_NETS:
        import lseg_b200  # noqa: F401
        from lseg_b200.lseg_net import LSegNet
        bb = OTHER[tag]["backbone"]
        n = LSegNet(labels=synth.ade20k_labels(), **{**NET_KW, "backbone": bb})
        n.load_state_dict(state_dict(0, bb))
        _OTHER_NETS.clear()  # one extra engine resident at a time (weights + plans ~ 3 GB each)
        _OTHER_NETS[tag] = n.cuda().eval()
    return _OTHER_NETS[tag]


@pytest.mark.parametrize("tag,B,H,W,K", [("b32", 2, 64, 96, 5), ("b32", 1, 480, 480, 150), ("b32", 3, 160, 224, 7),
                                         ("b32", 8, 480, 480, 150), ("rn50x16", 2, 64, 96, 5),
                                         ("rn50x16", 1, 480, 480, 150), ("rn50x16", 8, 480, 480, 150)])
def test_other_backbone_forward_vs_oracle(tag, B, H, W, K):
    from oracle import lseg_oracle as O
    cfg = OTHER[tag]
    bb, D, P = cfg["backbone"], cfg["D"], cfg["patch"]
    net_o = other_net(tag)
    labels = synth.ade20k_labels()[:K]
    tokens = synth.tokenize(labels)
    x = synth.make_image(B, H, W, seed=B * 1000 + H + 32)
    ref, st = O.lseg_forward(x, tokens, state_dict(0, bb), return_stages=True, backbone=bb)
    eng = net_o._engine_for(torch.device("cuda"))
    assert st["text_features"].shape[1] == eng.out_c == net_o.out_c
    got_tf = eng.forward(x.cuda(), _padded_text(eng, st["text_features"]), K)
    N = (H // P) * (W // P) + 1
    d = {"launches": eng.last_launch_count()}
    for k in range(4):
        tap = eng.debug_tensor(f"tap{k}", (B, N, D), torch.float32)
        d[f"tap{k}"] = rel_err(tap, st["taps"][k])
        lay = st["layers"][k]
        c, lh, lw = lay.shape[1], lay.shape[2], lay.shape[3]
        got_l = eng.debug_tensor(f"layer{k}", (B, lh, lw, cfg["stored"][k]), torch.float16).permute(0, 3, 1, 2).float()
        d[f"layer{k}"] = rel_err(got_l[:, :c], lay)
        d[f"layer{k}_tol"] = logit_tolerance(lay, STAGE_TOL)  # stored in fp16: the stage tolerance + one quantum
        d[f"layer{k}_pad_max"] = float(got_l[:, c:].abs().max()) if cfg["stored"][k] > c else 0.0
    p1 = eng.debug_tensor("path1", (B, H // 2, W // 2, 256), torch.float16)
    d["path1"] = rel_err(p1.permute(0, 3, 1, 2), st["path_1"])
    d["logits_teacher_forced"] = rel_err(got_tf, ref)
    d["logit_tol_tf"] = logit_tolerance(ref, LOGIT_REL)
    tf = argmax_report(got_tf, ref, margin_eps(ref, MARGIN_QUANTA_TF))
    d.update({"tf_" + k: v for k, v in tf.items()})
    got = net_o(x.cuda(), tokens)
    d["logits"] = rel_err(got, ref)
    # own text tower: TEXT_FLOOR_FACTOR x what the reference's own two executions of THIS backbone's fp16 text tower differ
    # by in the logits (recorded in the backbone's fixture by oracle/make_golden_backbones.py: 2.97e-3 for ViT-B/32, whose
    # max|logit| sits just above 1.0, 1.76e-3 for RN50x16), never below the default backbone's FULL_LOGIT_REL — the same
    # rule as test_other_backbone_against_reference_golden
    floor = float(np.load(os.path.join(GOLD, f"ref_{tag}.npz"))["k150_floor"])
    d["reference_floor"] = floor
    d["logit_tol_full"] = logit_tolerance(ref, max(FULL_LOGIT_REL, TEXT_FLOOR_FACTOR * floor))
    full = argmax_report(got, ref, margin_eps(ref))
    d.update(full)
    _report(f"{tag}_forward_B{B}_{H}x{W}_K{K}", d)
    assert torch.isfinite(got).all()
    for k in range(4):
        assert d[f"tap{k}"] <= STAGE_TOL and d[f"layer{k}"] <= d[f"layer{k}_tol"], d
        assert d[f"layer{k}_pad_max"] == 0.0, d  # the channel pad (96 -> 128) carries zero weights: exactly zero
    assert d["path1"] <= STAGE_TOL, d
    assert d["logits_teacher_forced"] <= d["logit_tol_tf"], d
    assert tf["ok"], d
    assert d["logits"] <= d["logit_tol_full"], d
    assert full["ok"], d


@pytest.mark.parametrize("tag", ["b32", "rn50x16"])
def test_other_backbone_against_reference_golden(tag):
    """Outputs of the UNMODIFIED reference LSegNet with that backbone (oracle/make_golden_backbones.py)."""
    net_o = other_net(tag)
    g = np.load(os.path.join(GOLD, f"ref_{tag}.npz"))
    labels = [str(s) for s in g["small_labels"]]
    x = synth.make_image(2, 64, 96, seed=2064)
    got = net_o(x.cuda(), synth.tokenize(labels)).cpu()
    ref = torch.from_numpy(g["small_logits"])
    # logits tolerance = TEXT_FLOOR_FACTOR x what the reference's own two executions of the fp16 text tower (the module
    # behind this fixture vs the oracle's recipe) differ by in THESE logits, recorded in the fixture, + one fp16 quantum;
    # never below the default backbone's FULL_LOGIT_REL
    rel_small = max(FULL_LOGIT_REL, TEXT_FLOOR_FACTOR * float(g["small_floor"]))
    rel_k150 = max(FULL_LOGIT_REL, TEXT_FLOOR_FACTOR * float(g["k150_floor"]))
    d = {"small_logits": rel_err(got, ref), "small_tol": logit_tolerance(ref, rel_small), "k150_floor": float(g["k150_floor"])}
    rep = argmax_report(got, ref, margin_eps(ref))
    x = synth.make_image(1, 480, 480, seed=1480)
    got = net_o(x.cuda(), synth.tokenize(synth.ade20k_labels())).cpu()
    lat = torch.from_numpy(g["k150_logits_lattice"])
    d["k150_lattice"] = rel_err(on_lattice(got, lat), lat)
    mask = torch.from_numpy(g["k150_argmax"].astype(np.int64))
    margin = torch.from_numpy(g["k150_margin_f16"].astype(np.float32))
    mism = got.argmax(1) != mask
    eps = MARGIN_QUANTA_FULL * fp16_quantum(lat.abs().max())
    d["k150_mismatch"] = int(mism.sum())
    d["k150_worst_mismatch_margin"] = float(margin[mism].max()) if d["k150_mismatch"] else 0.0
    d["margin_eps"] = eps
    _report(f"{tag}_reference_golden", d)
    assert d["small_logits"] <= d["small_tol"] and rep["ok"], (d, rep)
    assert d["k150_lattice"] <= logit_tolerance(lat, rel_k150), d
    assert d["k150_mismatch"] == 0 or d["k150_worst_mismatch_margin"] < eps, d


def test_forward_on_side_streams(net):
    """Everything a forward enqueues goes to the CALLER's current stream (no implicit legacy-stream work): issued on a
    non-default stream — default and highest priority — while another stream keeps the GPU busy, it returns the bits of
    the default-stream forward. Also the low-res entry point of the multi-GPU gather."""
    from lseg_b200 import ops
    tokens = synth.tokenize(synth.ade20k_labels()[:19])
    x = synth.make_image(3, 160, 224, seed=5).cuda()
    eng = net._engine_for(torch.device("cuda"))
    text = net._text_features(eng, tokens)
    ref = eng.forward(x, text, 19).clone()
    ref_lr = eng.forward_lowres(x, text, 19).clone()
    assert torch.equal(ops.upsample2x_nchw(ref_lr), ref)
    torch.cuda.synchronize()
    noise_stream = torch.cuda.Stream()
    junk = torch.randn(4096, 4096, device="cuda")
    prios = [0, -1]
    if hasattr(torch.cuda.Stream, "priority_range"):
        prios.append(torch.cuda.Stream.priority_range()[1])
    for prio in prios:
        s = torch.cuda.Stream(priority=prio)
        with torch.cuda.stream(noise_stream):
            for _ in range(20):
                junk = junk @ junk * 1e-4
        with torch.cuda.stream(s):
            out = eng.forward(x, text, 19)
            lr = eng.forward_lowres(x, text, 19)
            out2 = eng.forward(x, text, 19)
        s.synchronize()
        torch.cuda.synchronize()
        assert torch.equal(out, ref), prio
        assert torch.equal(lr, ref_lr), prio
        assert torch.equal(out2, ref), prio


# ------------------------------------------------------------------------------------------------
# LSegRNNetZS: the zero-shot model on the ResNet-101 trunk (lseg_net_zs.py:240-378, backbone "clip_resnet101")
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def net_rn():
    import lseg_b200  # noqa: F401
    from lseg_b200.lseg_net import LSegRNNetZS
    names = [line.strip() for line in open(os.path.join(GOLD, "fewshot_pascal.txt")) if line.strip()]
    n = LSegRNNetZS(label_list=names, features=256, arch_option=0, block_depth=0, activation="lrelu")
    n.load_state_dict(state_dict(0, "clip_resnet101"))
    return n.cuda().eval()


@pytest.mark.parametrize("B,H,W", [(3, 96, 128), (1, 480, 480), (8, 480, 480)])
def test_rn101_zs_forward_vs_oracle(net_rn, B, H, W):
    """ResNet stages (the fp16 operands of scratch.layerN_rn), path_1 and the zero-shot logits against the oracle; the
    stages and path_1 are stored in fp16: stage tolerance + one quantum. CPU emulation of the engine's rounding points
    (fp16 conv operands, fp32 residual stream) puts the stages at 0.6-0.7e-3."""
    from oracle import lseg_oracle as O
    sd = state_dict(0, "clip_resnet101")
    texts = [synth.tokenize(["others", n]) for n in net_rn.label_list]
    x = synth.make_image(B, H, W, seed=B * 1000 + H + 101)
    class_info = torch.tensor([(3 + 5 * i) % len(texts) for i in range(B)])
    ref, st = O.lseg_forward_rn_zs(x, class_info, texts, sd, return_stages=True)
    got = net_rn(x.cuda(), class_info)
    eng = net_rn._engine_for(torch.device("cuda"))
    d = {"launches": eng.last_launch_count()}
    for k in range(4):
        lay = st["layers"][k]
        c, lh, lw = lay.shape[1], lay.shape[2], lay.shape[3]
        got_l = eng.debug_tensor(f"layer{k}", (B, lh, lw, c), torch.float16).permute(0, 3, 1, 2).float()
        d[f"layer{k}"] = rel_err(got_l, lay)
        d[f"layer{k}_tol"] = logit_tolerance(lay, STAGE_TOL)
    p1 = eng.debug_tensor("path1", (B, H // 2, W // 2, 256), torch.float16)
    d["path1"] = rel_err(p1.permute(0, 3, 1, 2), st["path_1"])
    d["path1_tol"] = logit_tolerance(st["path_1"], STAGE_TOL)
    d["logits"] = rel_err(got, ref)
    d["logit_tol_full"] = logit_tolerance(ref, FULL_LOGIT_REL)
    full = argmax_report(got, ref, margin_eps(ref))
    d.update(full)
    _report(f"rn101_zs_forward_B{B}_{H}x{W}", d)
    assert got.shape == (B, 2, H, W) and torch.isfinite(got).all()
    for k in range(4):
        assert d[f"layer{k}"] <= d[f"layer{k}_tol"], d
    assert d["path1"] <= d["path1_tol"], d
    assert d["logits"] <= d["logit_tol_full"], d
    assert full["ok"], d
    assert torch.equal(net_rn.predict(x.cuda(), class_info), torch.max(got, 1)[1])


def test_rn101_zs_against_reference_golden(net_rn):
    """Outputs of the UNMODIFIED reference LSegRNNetZS (oracle/make_golden_rn.py)."""
    g = np.load(os.path.join(GOLD, "ref_rn101.npz"))
    x = synth.make_image(3, 96, 128, seed=77)
    got = net_rn(x.cuda(), torch.from_numpy(g["small_class_info"])).cpu()
    ref = torch.from_numpy(g["small_logits"])
    rel_small = max(FULL_LOGIT_REL, TEXT_FLOOR_FACTOR * float(g["small_floor"]))
    d = {"small_logits": rel_err(got, ref), "small_tol": logit_tolerance(ref, rel_small)}
    rep = argmax_report(got, ref, margin_eps(ref))
    x = synth.make_image(2, 480, 480, seed=1480)
    got = net_rn(x.cuda(), torch.from_numpy(g["s480_class_info"])).cpu()
    lat = torch.from_numpy(g["s480_logits_lattice"])
    rel_480 = max(FULL_LOGIT_REL, TEXT_FLOOR_FACTOR * float(g["s480_floor"]))
    d["s480_lattice"] = rel_err(on_lattice(got, lat), lat)
    mask = torch.from_numpy(g["s480_argmax"].astype(np.int64))
    margin = torch.from_numpy(g["s480_margin_f16"].astype(np.float32))
    mism = got.argmax(1) != mask
    eps = MARGIN_QUANTA_FULL * fp16_quantum(lat.abs().max())
    d["s480_mismatch"] = int(mism.sum())
    d["s480_worst_mismatch_margin"] = float(margin[mism].max()) if d["s480_mismatch"] else 0.0
    _report("rn101_reference_golden", d)
    assert d["small_logits"] <= d["small_tol"] and rep["ok"], (d, rep)
    assert d["s480_lattice"] <= logit_tolerance(lat, rel_480), d
    assert d["s480_mismatch"] == 0 or d["s480_worst_mismatch_margin"] < eps, d


def test_against_reference_golden(net):
    """The committed outputs of the UNMODIFIED reference modules (oracle/make_golden.py) at 480x480, K=150 and K=2:
    logits on the stored pixel lattice, full argmax mask, margins."""
    for tag, labels in (("k150", synth.ade20k_labels()), ("k2", ["cat", "other"])):
        g = np.load(os.path.join(GOLD, f"ref_480_{tag}.npz"))
        x = synth.make_image(1, 480, 480, seed=1480)
        got = net(x.cuda(), synth.tokenize(labels)).cpu()
        lat = torch.from_numpy(g["logits_lattice"])
        d = {"logits_lattice": rel_err(on_lattice(got, lat), lat)}
        mask = torch.from_numpy(g["argmax"].astype(np.int64))
        margin = torch.from_numpy(g["margin_f16"].astype(np.float32))
        mism = got.argmax(1) != mask
        eps = MARGIN_QUANTA_FULL * fp16_quantum(lat.abs().max())
        d["mismatch"] = int(mism.sum())
        d["worst_mismatch_margin"] = float(margin[mism].max()) if d["mismatch"] else 0.0
        d["margin_eps"] = eps
        _report(f"reference_golden_480_{tag}", d)
        assert d["logits_lattice"] <= logit_tolerance(lat, FULL_LOGIT_REL), d
        assert d["mismatch"] == 0 or d["worst_mismatch_margin"] < eps, d
        if tag == "k2":
            assert d["mismatch"] == 0, d


def test_predict_is_argmax_of_forward(net):
    """SURVEY 8(f) row 2 (fused argmax epilogue): predict() == torch.max(forward(), 1)[1], without the fp32 logits;
    checked against the unfused path bit for bit and against the oracle under the margin rule."""
    tokens = synth.tokenize(synth.ade20k_labels())
    x = synth.make_image(2, 480, 480, seed=9).cuda()
    logits = net(x, tokens)
    mask = net.predict(x, tokens)
    assert mask.dtype == torch.int64 and mask.shape == (2, 480, 480)
    assert torch.equal(mask.cpu(), torch.max(logits.cpu(), 1)[1])
    ref, _ = oracle_forward(x[:1].cpu(), tokens)
    rep = argmax_report_from_mask(mask[:1].cpu(), ref, margin_eps(ref))
    _report("predict_480_K150", rep)
    assert rep["ok"] and rep["agree_frac"] > 0.99, rep


def test_forward_rejects_bad_shapes(net):
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 473, 473, device="cuda"))
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 64, 64))  # CPU tensor: no fallback


# ------------------------------------------------------------------------------------------------
# BASELINE.json configs[3]: zero-shot path, PASCAL-5i / COCO-20i label files, 473x473
# ------------------------------------------------------------------------------------------------
def _label_file(name):
    return [line.strip() for line in open(os.path.join(GOLD, name)) if line.strip()]


def test_zero_shot_small():
    from lseg_b200.lseg_net import LSegNetZS
    from oracle import lseg_oracle as O
    names = _label_file("fewshot_pascal.txt")
    zs = LSegNetZS(label_list=names, **NET_KW)
    zs.load_state_dict(state_dict(0))
    zs = zs.cuda().eval()
    B, H, W = 3, 96, 96
    x = synth.make_image(B, H, W, seed=77)
    class_info = torch.tensor([3, 0, 17])
    texts = [synth.tokenize(["others", n]) for n in names]
    ref = O.lseg_forward_zs(x, class_info, texts, state_dict(0))
    got = zs(x.cuda(), class_info.cuda())
    d = {"logits": rel_err(got, ref)}
    d.update(argmax_report(got, ref, margin_eps(ref)))
    gold = np.load(os.path.join(GOLD, "ref_zs.npz"))  # the unmodified reference LSegNetZS on the same inputs
    d["logits_vs_reference_golden"] = rel_err(got, torch.from_numpy(gold["logits"]))
    _report("zero_shot_B3_96", d)
    assert got.shape == (B, 2, H, W)
    assert d["logits"] <= logit_tolerance(ref, FULL_LOGIT_REL) and d["ok"], d
    assert d["logits_vs_reference_golden"] <= logit_tolerance(ref, FULL_LOGIT_REL), d


@pytest.mark.parametrize("label_file", ["fewshot_pascal.txt", "fewshot_coco.txt"])
def test_zero_shot_config4(label_file):
    """configs[3]: B=8 images of 473x473. 473 is not runnable by the reference ViT path (token grid 29.56; the reference's
    own ZS script evaluates at 480, test_lseg_zs.py:268-270), so the input is padded to 480 with the normalised zero
    value -1 exactly like pad_image (additional_utils/models.py:145-156) and the output is cropped back — on both sides."""
    from lseg_b200.lseg_net import LSegNetZS
    from oracle import lseg_oracle as O
    names = _label_file(label_file)
    zs = LSegNetZS(label_list=names, **NET_KW)
    zs.load_state_dict(state_dict(0))
    zs = zs.cuda().eval()
    B = 8
    x473 = synth.make_image(B, 473, 473, seed=473)
    x = F.pad(x473, (0, 7, 0, 7), value=-1.0)
    g = torch.Generator().manual_seed(4)
    class_info = torch.randint(0, len(names), (B,), generator=g)
    texts = [synth.tokenize(["others", n]) for n in names]
    ref = O.lseg_forward_zs(x, class_info, texts, state_dict(0))[:, :, :473, :473]
    got = zs(x.cuda(), class_info.cuda())[:, :, :473, :473]
    mask = zs.predict(x.cuda(), class_info.cuda())[:, :473, :473]
    d = {"logits": rel_err(got, ref), "n_classes": len(names)}
    d.update(argmax_report(got, ref, margin_eps(ref)))
    _report(f"zero_shot_cfg4_{label_file.split('.')[0]}", d)
    assert got.shape == (B, 2, 473, 473)
    assert torch.equal(mask.cpu(), got.argmax(1).cpu())
    assert d["logits"] <= logit_tolerance(ref, FULL_LOGIT_REL) and d["ok"], d


# ------------------------------------------------------------------------------------------------
# BASELINE.json configs[4]: open-vocabulary stress, 720x720, 512 synthetic prompts
# ------------------------------------------------------------------------------------------------
def test_open_vocab_config5(net):
    """configs[4] at B=1: 720 is not runnable (odd 45-token grid: the reference raises a 46-vs-45 size mismatch), so the
    image is padded to 736 with -1 (pad_image) and the logits are cropped back to 720 — stated, and done on both sides.
    N = 2117 tokens (34 key tiles, 17 query tiles of the attention kernel), K = 512 = 4 weight tiles of the pixel x text
    GEMM, 135 424 pixels."""
    tokens = synth.synthetic_prompts(512, seed=0)
    x720 = synth.make_image(1, 720, 720, seed=720)
    x = F.pad(x720, (0, 16, 0, 16), value=-1.0)
    ref, st = oracle_forward(x, tokens)
    eng = net._engine_for(torch.device("cuda"))
    got_tf = eng.forward(x.cuda(), _padded_text(eng, st["text_features"]), 512)[:, :, :720, :720]
    got = net(x.cuda(), tokens)[:, :, :720, :720]
    ref = ref[:, :, :720, :720]
    d = {"logits_teacher_forced": rel_err(got_tf, ref), "logits": rel_err(got, ref),
         "max_abs_logit": ref.abs().max().item()}
    tf = argmax_report(got_tf, ref, margin_eps(ref, MARGIN_QUANTA_TF))
    d.update({"tf_" + k: v for k, v in tf.items()})
    d.update(argmax_report(got, ref, margin_eps(ref)))
    N = 46 * 46 + 1
    for k in range(4):
        d[f"tap{k}"] = rel_err(eng.debug_tensor(f"tap{k}", (1, N, 1024), torch.float32), st["taps"][k])
    _report("open_vocab_cfg5_736_K512", d)
    for k in range(4):
        assert d[f"tap{k}"] <= STAGE_TOL, d
    assert d["logits_teacher_forced"] <= logit_tolerance(ref, LOGIT_REL) and tf["ok"], d
    assert d["logits"] <= logit_tolerance(ref, FULL_LOGIT_REL) and d["ok"], d


@pytest.mark.parametrize("tag,kw", [("opt1", dict(arch_option=1, block_depth=2, activation="lrelu")),
                                    ("opt2", dict(arch_option=2, block_depth=3, activation="tanh"))])
def test_arch_option_head_blocks(tag, kw):
    """arch_option 1 / 2 (SURVEY 8(a) row a16; lseg_net.py:148-154,198-201) against the oracle AND against the committed
    output of the unmodified reference LSegNet (oracle/make_golden_arch.py). The blocks themselves are exact to 2e-6
    (tests/test_ops_gpu.py::test_head_block, tests/test_oracle.py bit-level vs the reference module); what this case
    measures end to end is how much they AMPLIFY the upstream differences (shared 3x3 taps up to 0.4 and a channel max,
    applied block_depth times: x3-4 per application), hence the wider bar."""
    from lseg_b200.lseg_net import LSegNet
    from oracle import lseg_oracle as O
    sd = synth.make_state_dict(0, head_block=True)
    labels = synth.ade20k_labels()[:5]
    nk = dict(NET_KW)
    nk.update(kw)
    n = LSegNet(labels=labels, **nk)
    n.load_state_dict(sd)
    n = n.cuda().eval()
    x = synth.make_image(2, 64, 96, seed=2064)
    tokens = synth.tokenize(labels)
    ref, st = O.lseg_forward(x, tokens, sd, return_stages=True, **kw)
    eng = n._engine_for(torch.device("cuda"))
    got_tf = eng.forward(x.cuda(), _padded_text(eng, st["text_features"]), 5)
    got = n(x.cuda(), tokens)
    mask = n.predict(x.cuda(), tokens)
    gold = np.load(os.path.join(GOLD, "ref_arch.npz"))
    d = {"logits_teacher_forced": rel_err(got_tf, ref), "logits": rel_err(got, ref),
         "logits_vs_reference_golden": rel_err(got, torch.from_numpy(gold[f"{tag}_logits"])),
         "max_abs_logit": ref.abs().max().item()}
    _report(f"arch_option_{tag}", d)
    assert torch.equal(mask.cpu(), got.argmax(1).cpu())  # fused argmax reads the same fp32 block output
    assert d["logits_teacher_forced"] <= 6e-3, d
    assert d["logits"] <= 2e-2 and d["logits_vs_reference_golden"] <= 2e-2, d


def test_argmax_planted_prototypes(net):
    """Argmax parity with well-separated classes. Random text embeddings give near-tie logits almost
    everywhere (SURVEY.md section 7), so this case plants K=150 class prototypes: the oracle's own
    normalised pixel embeddings at seeded pixel positions are used as 'text features'. Every pixel then has
    a clear winner, and the image trunk + head + correlation + upsample must reproduce the oracle's mask."""
    from oracle import lseg_oracle as O
    sd = state_dict(0)
    B, H, W, K = 1, 480, 480, 150
    x = synth.make_image(B, H, W, seed=1480)
    layers = O.forward_vit(x, sd)
    path_1 = O.decoder(layers, sd)
    feat = F.conv2d(path_1, sd["scratch.head1.weight"], sd["scratch.head1.bias"])
    feat = feat.permute(0, 2, 3, 1).reshape(-1, 512)
    g = torch.Generator().manual_seed(11)
    idx = torch.randperm(feat.shape[0], generator=g)[:K]
    # random-weight pixel embeddings share one dominant direction (cos to the mean ~0.99), so the prototypes
    # are centred: classes are then separated by the per-pixel deviation (oracle margins > 0.5 for 99% of pixels)
    protos = feat[idx] - feat.mean(dim=0, keepdim=True)
    protos = (protos / protos.norm(dim=-1, keepdim=True)).half()
    ref = O.output_conv(O.correlation_head(path_1, protos, sd))
    eng = net._engine_for(torch.device("cuda"))
    got = eng.forward(x.cuda(), _padded_text(eng, protos), K)
    d = {"logits": rel_err(got, ref), "max_abs_logit": ref.abs().max().item()}
    d.update(argmax_report(got, ref, margin_eps(ref, MARGIN_QUANTA_TF)))
    _report("planted_prototypes_480_K150", d)
    assert d["logits"] <= LOGIT_REL, d  # real margins, large logits: the plain 1e-3 holds
    assert d["ok"] and d["agree_frac"] > 0.9999, d


def test_batch_consistency(net):
    """Size-independent property at the bench size: images are independent (eval-mode BN). In deterministic mode
    (the default: fixed summation order) a batch-8 forward equals a batch-1 forward bit for bit; with split-K
    allowed the residual GEMMs may split K differently for the two batch sizes, which moves fp32 roundings only."""
    from lseg_b200 import ops
    tokens = synth.tokenize(["cat", "other", "tree"])
    x = synth.make_image(8, 480, 480, seed=5).cuda()
    ops.set_deterministic(True)
    try:
        full = net(x, tokens)
        one = net(x[3:4].contiguous(), tokens)
        assert torch.equal(full[3:4].argmax(1), one.argmax(1))
        assert (full[3:4] - one).abs().max().item() == 0.0
        again = net(x, tokens)
        assert torch.equal(full, again)  # run-to-run reproducible
        ops.set_deterministic(False)  # split-K allowed: same numbers up to fp32 summation order
        fast = net(x, tokens)
        one_fast = net(x[3:4].contiguous(), tokens)
        scale = full.abs().max().item()
        assert (fast - full).abs().max().item() <= 2e-3 * scale
        assert (fast[3:4] - one_fast).abs().max().item() <= 2e-3 * scale
    finally:
        ops.set_deterministic(True)
