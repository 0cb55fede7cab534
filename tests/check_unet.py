"""GPU parity of the CUDA UNet (fwd + bwd) against the fp32 CPU oracle on a tiny SD-style config.

usage: python tests/check_unet.py [plain|v1|v2|v1_stacked|v1_post_add|v1_concat|none] ...   (default: all, each in a subprocess)
"""
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tests._device import DEV  # noqa: E402  ("cuda", or "cpu" in the emulated host-logic mode)

TINY = dict(block_out_channels=(64, 128, 128, 128), layers_per_block=1, cross_attention_dim=64, attention_head_dim=8)
TINY_LORA = dict(
    lora_block_out_channels=(64, 128, 128, 128),
    lora_cross_attention_dims=([None, 64] * 3, [None, 64] * 3, [None, 64] * 3, [None, 64]),
)


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def build_pair(variant, B=2, HW=16, seed=0):
    import torch
    from oracle import models_ref as MR
    from oracle import unet_ref as UR
    import controllora_b200 as cb

    torch.manual_seed(seed)
    ounet = UR.UNet2DConditionModel(**TINY)
    UR.init_synthetic_(ounet, seed=1)
    # the frozen network runs in bf16 in the reference: round the oracle's weights so both sides share them exactly
    with torch.no_grad():
        for p in ounet.parameters():
            p.copy_(p.to(torch.bfloat16).float())
    sd = {k: v.detach().clone() for k, v in ounet.state_dict().items()}
    munet = cb.UNet2DConditionModel.from_state_dict(sd, DEV, TINY)

    kw = dict(TINY_LORA)
    if variant == "v2":
        kw.update(lora_control_version=2, lora_pre_conv_skipped=True)
    if variant == "v1_post_add":
        kw.update(lora_post_add=True)            # configs/post-add.json: every adapter reads its projection's output
    if variant == "v1_concat":
        # configs/danbooru-sketch.json flavour: to_control = MLP over [h ; c] with a control rank well above the LoRA rank
        kw.update(lora_concat_hidden=True, lora_control_rank=32, lora_pre_conv_skipped=True, lora_control_self_add=False)
    ocl = MR.ControlLoRA(**kw) if variant != "none" else None
    mcl = cb.ControlLoRA(**kw) if variant != "none" else None
    if ocl is not None:
        MR.randomize_lora_up_(ocl, seed=3, std=0.05)
        mcl.load_state_dict(ocl.state_dict())
        mcl.to(DEV)
        if variant == "plain":
            # plain LoRACrossAttnProcessor on every layer (the DreamBooth-LoRA / pre_lora flavour)
            oprocs, mprocs = {}, {}
            g = torch.Generator().manual_seed(7)
            for name in ounet.attn_processors.keys():
                oa = dict(ounet._attn_modules())[name]
                C = oa.to_q.weight.shape[0]
                xd = None if name.endswith("attn1.processor") else TINY["cross_attention_dim"]
                op = MR.LoRACrossAttnProcessor(C, xd, rank=4)
                for n_, p_ in op.named_parameters():
                    if n_.endswith("up.weight"):
                        with torch.no_grad():
                            p_.copy_(0.05 * torch.randn(p_.shape, generator=g))
                mp = cb.LoRACrossAttnProcessor(C, xd, rank=4)
                mp.load_state_dict(op.state_dict())
                oprocs[name], mprocs[name] = op, mp.to(DEV)
            ounet.set_attn_processor(oprocs)
            munet.set_attn_processor(mprocs)
        else:
            oprocs = MR.wire_processors(ounet, ocl)
            mprocs = MR.wire_processors(munet, mcl)
            if variant == "v1_stacked":
                g = torch.Generator().manual_seed(11)
                for name in oprocs:
                    C = oprocs[name].hidden_size
                    xd = oprocs[name].cross_attention_dim
                    op = MR.LoRACrossAttnProcessor(C, xd, rank=4)
                    for n_, p_ in op.named_parameters():
                        if n_.endswith("up.weight"):
                            with torch.no_grad():
                                p_.copy_(0.05 * torch.randn(p_.shape, generator=g))
                    mp = cb.LoRACrossAttnProcessor(C, xd, rank=4).to(DEV)
                    mp.load_state_dict(op.state_dict())
                    oprocs[name].inject_pre_lora(op)
                    mprocs[name].inject_pre_lora(mp)
                    oprocs[name]._extra = op
                    mprocs[name]._extra = mp
    return ounet, munet, ocl, mcl


def run(variant):
    """variant[@scale]: e.g. "v1_stacked@0.5" runs with cross_attention_kwargs={"scale": 0.5} (models.py:118-120: the
    processors' `scale` argument; stacked value adapters stay unscaled, models.py:260,265,397,402)."""
    import torch
    from oracle import models_ref as MR

    torch.backends.cuda.matmul.allow_tf32 = False
    B, HW = 2, 16
    scale = 1.0
    if "@" in variant:
        variant, sc = variant.split("@")
        scale = float(sc)
    cak = None if scale == 1.0 else {"scale": scale}
    ounet, munet, ocl, mcl = build_pair(variant, B, HW)
    g = torch.Generator().manual_seed(5)
    sample = torch.randn(B, 4, HW, HW, generator=g).to(torch.bfloat16).float()
    t = torch.tensor([17, 801])
    ehs = torch.randn(B, 77, TINY["cross_attention_dim"], generator=g).to(torch.bfloat16).float()
    target = torch.randn(B, 4, HW, HW, generator=g)
    ch = TINY["block_out_channels"]
    ctrl_o, ctrl_m = [], []
    if variant in ("v1", "v1_stacked", "v2", "v1_post_add", "v1_concat"):
        cc = [256] * 4 if variant in ("v2", "v1_concat") else list(ch)
        for lvl in range(4):
            s = HW >> lvl
            c = (0.5 * torch.randn(B, cc[lvl], s, s, generator=g)).to(torch.bfloat16).float()
            co = c.clone().requires_grad_(True)
            cm = c.clone().to(DEV).requires_grad_(True)
            ctrl_o.append(co)
            ctrl_m.append(cm)
            for p in ocl.lora_layers[lvl]:
                p.inject_control_states(co)
            for p in mcl.lora_layers[lvl]:
                p.inject_control_states(cm)
    # ---- oracle (CPU, fp32)
    t0 = time.time()
    po = ounet(sample, t, ehs, cross_attention_kwargs=cak).sample
    lo = torch.nn.functional.mse_loss(po, target)
    oparams = {}
    if variant != "none":
        lo.backward()
    label = variant if scale == 1.0 else f"{variant}@{scale}"
    print(f"[{label}] oracle fwd+bwd {time.time()-t0:.1f}s  loss={float(lo):.6f}")
    # ---- ours
    pm = munet(sample.to(DEV), t.to(DEV), ehs.to(DEV).to(torch.bfloat16), cross_attention_kwargs=cak).sample
    lm = torch.nn.functional.mse_loss(pm, target.to(DEV))
    if variant != "none":
        lm.backward()
    if DEV == "cuda":
        torch.cuda.synchronize()
    e_pred = rel(pm, po)
    print(f"[{label}] noise-pred rel={e_pred:.3e}  loss ours={float(lm):.6f}")
    worst = 0.0
    if variant != "none":
        # parameters: match by traversal order of the processors
        onames = list(ounet.attn_processors.keys())
        rows = []
        for name in onames:
            op, mp = ounet.attn_processors[name], munet.attn_processors[name]
            pairs = [(op, mp)]
            if hasattr(op, "_extra"):
                pairs.append((op._extra, mp._extra))
            for o_, m_ in pairs:
                for (n1, p1), (n2, p2) in zip(o_.named_parameters(), m_.named_parameters()):
                    assert n1 == n2
                    if p1.grad is None:
                        continue
                    assert p2.grad is not None, (name, n2)
                    e = rel(p2.grad, p1.grad)
                    rows.append((e, name, n1, float(p1.grad.norm())))
        rows.sort(reverse=True)
        for e, name, n1, nrm in rows[:8]:
            print(f"    grad rel={e:.3e} |g|={nrm:.3e} {name} {n1}")
        worst = rows[0][0]
        allg_o = torch.cat([ounet.attn_processors[n].get_parameter(k).grad.flatten() for n in onames
                            for k, _ in ounet.attn_processors[n].named_parameters()
                            if ounet.attn_processors[n].get_parameter(k).grad is not None])
        allg_m = torch.cat([munet.attn_processors[n].get_parameter(k).grad.flatten().cpu() for n in onames
                            for k, _ in munet.attn_processors[n].named_parameters()
                            if ounet.attn_processors[n].get_parameter(k).grad is not None])
        print(f"[{label}] all LoRA grads (concatenated) rel={rel(allg_m, allg_o):.3e}  worst tensor rel={worst:.3e}  n={len(rows)}")
        for lvl, (co, cm) in enumerate(zip(ctrl_o, ctrl_m)):
            print(f"    d control[{lvl}] rel={rel(cm.grad, co.grad):.3e} |g|={float(co.grad.norm()):.3e}")
    ok = e_pred < 2e-2 and worst < 8e-2
    print("CASE_OK" if ok else "CASE_FAIL")
    return ok


def main():
    variants = sys.argv[1:] or ["none", "plain", "v1", "v1_stacked", "v2"]
    if len(variants) == 1:
        sys.exit(0 if run(variants[0]) else 1)
    res = {}
    for v in variants:
        try:
            r = subprocess.run([sys.executable, __file__, v], capture_output=True, text=True, timeout=600)
            ok = r.returncode == 0 and "CASE_OK" in r.stdout
            out = r.stdout + r.stderr
        except subprocess.TimeoutExpired as e:
            ok, out = False, f"TIMEOUT {e}"
        res[v] = ok
        print(f"=== {v}: {'PASS' if ok else 'FAIL'}")
        lines = [l for l in out.strip().splitlines() if "Warning" not in l]
        for line in (lines if ok else lines[-40:]):
            print("    " + line)
        sys.stdout.flush()
    print("SUMMARY", res)


if __name__ == "__main__":
    main()
