"""Full-size parity and the precision contract at the SD-2-base shapes (tests/check_fullsize.py's contract, new row).

The SD-2 UNet (SD21_CONFIG: 320/640/1280/1280 channels with 5/10/20/20 heads of 64, linear projections, 77x1024 text states)
at 64x64 latents with a 512x512 guide, a named ControlLoRA config with its cross-attention adapters at 1024, and a
v-prediction target sqrt(a_t) noise - sqrt(1 - a_t) x0 (the SD-2.1 training loss).  Three arms run the same training-step
front half -- hint encoder, UNet, MSE, backward -- on the same seeded inputs and bf16-rounded weights:

  (o) the fp32 oracle on the CPU (oracle/unet_ref.py with tests/sd2_ref.py's per-block heads, oracle/models_ref.py)
  (a) ours, through the drop-in classes (the UNet loaded from the linear-projection state dict an SD-2 checkpoint holds)
  (b) the oracle code in eager PyTorch on the GPU at the reference's precision: bf16 UNet, fp32 adapters, bf16 autocast

and asserts err(a vs o) <= err(b vs o) for the noise prediction and the concatenated gradient of every trainable parameter,
with check_fullsize.py's absolute caps on the prediction, the gradient and the loss.

usage: python tests/check_fullsize_sd2.py [diffusiondb-canny-v2|diffusiondb-canny] [B]"""
import copy
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from tests.check_fullsize import CAP_GRAD_ALL, CAP_LOSS, CAP_PRED, MARGIN, rel, zero_grad_biases  # noqa: E402


def _inputs(torch, B, xd, ac):
    g = lambda s: torch.Generator().manual_seed(s)
    x0 = torch.randn(B, 4, 64, 64, generator=g(0))
    noise = torch.randn(B, 4, 64, 64, generator=g(5))
    t = torch.randint(0, 1000, (B,), generator=g(1))
    e = torch.randn(B, 77, xd, generator=g(2)).to(torch.bfloat16).float()
    edge = (torch.rand(B, 1, 512, 512, generator=g(3)) < 0.08).float() * 2 - 1
    shape = (-1, 1, 1, 1)
    sa, sb = ac[t].sqrt().view(shape), (1 - ac[t]).sqrt().view(shape)
    x = (sa * x0.double() + sb * noise.double()).float().to(torch.bfloat16).float()
    tgt = (sa * noise.double() - sb * x0.double()).float()
    return x, t, e, edge.expand(B, 3, 512, 512).contiguous(), tgt


def run(config_name="diffusiondb-canny-v2", B=1):
    import torch

    import controllora_b200 as cb
    from controllora_b200.configs import NAMED, wire_processors
    from controllora_b200.unet import SD21_CONFIG
    from oracle import models_ref as MR
    from oracle import sampler_ref as SR
    from oracle import unet_ref as UR
    from tests import sd2_ref as R

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = "cuda"
    xd = SD21_CONFIG["cross_attention_dim"]
    ccfg = dict(NAMED[config_name], lora_cross_attention_dims=([None, xd] * 5, [None, xd] * 5, [None, xd] * 5, [None, xd]))

    ounet = R.unet(SD21_CONFIG)
    UR.init_synthetic_(ounet, seed=1)
    with torch.no_grad():
        for p in ounet.parameters():
            p.copy_(p.to(torch.bfloat16).float())
    ounet.requires_grad_(False)
    ocl = MR.ControlLoRA.from_config(ccfg)
    MR.randomize_lora_up_(ocl, seed=3, std=0.02)
    g = torch.Generator().manual_seed(2)
    with torch.no_grad():
        for n, p in ocl.named_parameters():
            if "norm" in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
    bunet_cpu, bcl_cpu = copy.deepcopy(ounet), copy.deepcopy(ocl)
    MR.wire_processors(ounet, ocl)
    x, t, e, guide, tgt = _inputs(torch, B, xd, SR.alphas_cumprod())

    def arm_oracle(unet, cl, device, autocast):
        xs, ts, es, gs, tg = (v.to(device) for v in (x, t, e, guide, tgt))
        cl.zero_grad(set_to_none=True)
        if autocast:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                cl(gs)
                pred = unet(xs.to(torch.bfloat16), ts.long(), es.to(torch.bfloat16)).sample
                loss = torch.nn.functional.mse_loss(pred.float(), tg)
        else:
            cl(gs)
            pred = unet(xs, ts.long(), es).sample
            loss = torch.nn.functional.mse_loss(pred, tg)
        loss.backward()
        grads = {n: p.grad.detach().float().cpu().clone() for n, p in cl.named_parameters() if p.grad is not None}
        return pred.detach().float().cpu(), float(loss), grads

    # (a) ours
    sd = R.to_linear_projection({k: v.detach().clone() for k, v in ounet.state_dict().items() if "processor" not in k})
    munet = cb.UNet2DConditionModel.from_state_dict(sd, dev, SD21_CONFIG)
    mcl = cb.ControlLoRA.from_config(ccfg)
    mcl.load_state_dict(ocl.state_dict())
    mcl.to(dev)
    wire_processors(munet, mcl)
    mcl(guide.to(dev))
    pm = munet(x.to(dev), t.to(dev), e.to(dev).to(torch.bfloat16)).sample
    lm = torch.nn.functional.mse_loss(pm.float(), tgt.to(dev))
    lm.backward()
    torch.cuda.synchronize()
    pred_a, loss_a = pm.detach().float().cpu(), float(lm)
    grads_a = {n: p.grad.detach().float().cpu().clone() for n, p in mcl.named_parameters() if p.grad is not None}
    del munet, mcl, pm, lm, sd
    torch.cuda.empty_cache()

    # (o) fp32 oracle on the host
    t0 = time.time()
    pred_o, loss_o, grads_o = arm_oracle(ounet, ocl, "cpu", False)
    oracle_s = time.time() - t0

    # (b) eager bf16 on the GPU
    bunet = bunet_cpu.to(dev).to(torch.bfloat16)
    bcl = bcl_cpu.to(dev)
    MR.wire_processors(bunet, bcl)
    pred_b, loss_b, grads_b = arm_oracle(bunet, bcl, dev, True)
    del bunet, bcl
    torch.cuda.empty_cache()

    zero_b = zero_grad_biases(ocl)
    names = [n for n in grads_o if n not in zero_b]
    missing = [n for n in names if n not in grads_a]
    assert not missing, f"ours produced no gradient for {missing[:5]}"
    cat = lambda gr, sel: torch.cat([gr[n].flatten() for n in sel])
    res = {"pred": (rel(pred_a, pred_o), rel(pred_b, pred_o)),
           "loss": (abs(loss_a - loss_o) / abs(loss_o), abs(loss_b - loss_o) / abs(loss_o)),
           "grad_all": (rel(cat(grads_a, names), cat(grads_o, names)), rel(cat(grads_b, names), cat(grads_o, names)))}
    groups = {"hint_encoder": lambda n: not n.startswith("lora_layers"),
              "lora_adapters": lambda n: n.startswith("lora_layers") and "to_control" not in n,
              "control": lambda n: n.startswith("lora_layers") and "to_control" in n}
    for gname, fn in groups.items():
        sel = [n for n in names if fn(n)]
        if sel:
            res["grad_" + gname] = (rel(cat(grads_a, sel), cat(grads_o, sel)), rel(cat(grads_b, sel), cat(grads_o, sel)))
    print(f"== SD-2-base full-size parity: {config_name}, B={B}, v target; oracle fp32 CPU {oracle_s:.1f}s", flush=True)
    print(f"   loss: oracle {loss_o:.6f}  ours {loss_a:.6f}  eager-bf16 {loss_b:.6f}", flush=True)
    for k, (ea, eb) in res.items():
        print(f"   {k:<18} ours {ea:10.3e}   eager-bf16 {eb:10.3e}   ratio {ea / max(eb, 1e-30):5.2f}", flush=True)
    ok = all(res[k][0] <= MARGIN * res[k][1] for k in ("pred", "grad_all"))
    ok = ok and res["pred"][0] <= CAP_PRED and res["grad_all"][0] <= CAP_GRAD_ALL and res["loss"][0] <= CAP_LOSS
    print("   JSON " + json.dumps({"config": config_name, "batch": B, "ok": bool(ok),
                                   **{k: {"ours": v[0], "eager_bf16": v[1]} for k, v in res.items()}}), flush=True)
    return ok


if __name__ == "__main__":
    name = sys.argv[1] if len(sys.argv) > 1 else "diffusiondb-canny-v2"
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    sys.exit(0 if run(name, B) else 1)
