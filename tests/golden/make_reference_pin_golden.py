"""Generates tests/golden/reference_pin.pt: what the reference's own models.py computes (imported unmodified,
tests/golden/reference_import.py) in the cases of tests/test_reference_pin.py - the hint encoder of every shipped config, every
processor wiring, and the whole tiny UNet with the reference's processors.  Each case is one program below, run once with the
reference's classes (here, to write the file) and once with the restatement oracle/models_ref.py (in the test), on weights seeded
through the oracle classes (identical state-dict layout) and seeded inputs.  Tensors are kept as a fixed, seeded sample of at most
PIN_SAMPLE elements plus their full absolute maximum, which keeps the file small.

    python -m tests.golden.make_reference_pin_golden          (needs the reference tree)
"""
import contextlib
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import models_ref as MR  # noqa: E402
from oracle import unet_ref as UR  # noqa: E402
from tests.golden.make_reference_golden import sample_index  # noqa: E402

OUT = Path(__file__).resolve().parent / "reference_pin.pt"
CONFIGS = ["base", "fill50k", "diffusiondb-canny", "mpii-pose", "diffusiondb-canny-v2", "mpii-pose-v2", "post-add", "danbooru-sketch"]
PROC_CASES = {
    "plain_self": ("LoRACrossAttnProcessor", False, {}, None, 1.0),
    "plain_cross_post_add": ("LoRACrossAttnProcessor", True, dict(post_add=True), None, 0.7),
    "plain_skips": ("LoRACrossAttnProcessor", True, dict(key_states_skipped=True, output_states_skipped=True), None, 1.0),
    "v1_self": ("ControlLoRACrossAttnProcessor", False, {}, None, 1.0),
    "v1_cross_scale": ("ControlLoRACrossAttnProcessor", True, dict(control_rank=8), None, 0.5),
    "v1_post_add": ("ControlLoRACrossAttnProcessor", False, dict(post_add=True), None, 1.0),
    "v1_concat": ("ControlLoRACrossAttnProcessor", True, dict(concat_hidden=True, control_rank=16, control_channels=96), None, 1.0),
    "v1_stacked_pre_post": ("ControlLoRACrossAttnProcessor", True, {}, "plain", 0.5),
    "v1_stacked_control": ("ControlLoRACrossAttnProcessor", False, {}, "control", 0.8),
    "v2_self": ("ControlLoRACrossAttnProcessorV2", False, dict(control_channels=96), None, 1.0),
    "v2_cross_scale": ("ControlLoRACrossAttnProcessorV2", True, dict(control_channels=96, control_rank=8), None, 0.6),
    "v2_stacked": ("ControlLoRACrossAttnProcessorV2", False, dict(control_channels=96), "plain", 1.0),
    "v2_stacked_control": ("ControlLoRACrossAttnProcessorV2", True, dict(control_channels=96), "control", 0.9),
}
UNET_VARIANTS = ["v1", "v2", "post_add", "concat"]


PIN_SAMPLE = 32
_FULL = [False]


@contextlib.contextmanager
def full_tensors():
    """Inside: `summ` keeps every element (for comparisons where both sides run live)."""
    _FULL[0] = True
    try:
        yield
    finally:
        _FULL[0] = False


def summ(t):
    """A tensor as (fixed seeded sample of at most PIN_SAMPLE elements - all of them inside full_tensors() -, full shape, full
    absolute maximum)."""
    t = t.detach().float()
    shape = tuple(t.shape)
    t = t.reshape(-1)
    s = t.clone() if _FULL[0] else t[sample_index(t.numel())[:PIN_SAMPLE]].clone()
    return {"s": s, "shape": shape, "amax": float(t.abs().max()) if t.numel() else 0.0}


def pack(obj, buf):
    """Replace every sample tensor by its (offset, length) in one flat list `buf` (one tensor instead of thousands)."""
    if isinstance(obj, dict):
        if "s" in obj and isinstance(obj["s"], torch.Tensor):
            off = len(buf)
            buf.extend(obj["s"].tolist())
            return dict(obj, s=(off, obj["s"].numel()))
        return {k: pack(v, buf) for k, v in obj.items()}
    if isinstance(obj, list):
        return [pack(v, buf) for v in obj]
    return obj


def unpack(obj, flat):
    if isinstance(obj, dict):
        if "s" in obj and isinstance(obj["s"], tuple):
            off, k = obj["s"]
            return dict(obj, s=flat[off:off + k])
        return {k: unpack(v, flat) for k, v in obj.items()}
    if isinstance(obj, list):
        return [unpack(v, flat) for v in obj]
    return obj


def load():
    """The golden dictionary with every sample restored as a tensor."""
    gold = torch.load(OUT, weights_only=False)
    return unpack(gold["cases"], gold["flat"])


def randomize_(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("up.weight"):
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            elif "norm" in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))


def seeded(cls_name, *args, seed, **kw):
    """State dict of an oracle module of class `cls_name`, default-initialised under torch seed `seed` and randomised."""
    torch.manual_seed(seed)
    m = getattr(MR, cls_name)(*args, **kw)
    randomize_(m, seed + 1)
    return m.state_dict()


def build(M, cls_name, *args, sd, **kw):
    m = getattr(M, cls_name)(*args, **kw)
    m.load_state_dict(sd)
    return m


def run_hint(M, cfg):
    """ControlLoRA.__init__ wiring + forward / backward (models.py:618-835) of module M's class on the seeded weights."""
    torch.set_num_threads(1)
    cl = build(M, "ControlLoRA", sd=seeded("ControlLoRA", seed=0, **cfg), **cfg)
    attrs = ("hidden_size", "cross_attention_dim", "rank", "post_add", "concat_hidden", "control_self_add",
             "key_states_skipped", "value_states_skipped", "output_states_skipped")
    g = torch.Generator().manual_seed(2)
    guide = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    states = cl(guide).control_states
    ws = [torch.randn(s.shape, generator=g) for s in states]
    sum((s * w).sum() for s, w in zip(states, ws)).backward()
    return {"keys": list(cl.state_dict().keys()),
            "types": [[type(p).__name__ for p in lvl] for lvl in cl.lora_layers],
            "attrs": [[getattr(p, a) for a in attrs] for lvl in cl.lora_layers for p in lvl],
            "states": [summ(s) for s in states],
            "grads": {n: (None if p.grad is None else summ(p.grad)) for n, p in cl.named_parameters()},
            # the processors received the injected tensors (models.py:826-829)
            "injected": [[tuple(p.control_states.shape) == tuple(s.shape) and bool(torch.equal(p.control_states, s)) for p in lvl]
                         for lvl, s in zip(cl.lora_layers, states)]}


def run_processor(M, case):
    """One processor call (models.py:118-152 / 222-287 / 357-431) of module M's classes on a shared attention module: output,
    d hidden, every parameter gradient, d control."""
    torch.set_num_threads(1)
    cls, cross, kw, stack, scale = PROC_CASES[case]
    C, XD, H = 64, 48, 4
    xd = XD if cross else None
    torch.manual_seed(3)
    attn = UR.CrossAttention(C, xd, H, C // H)
    proc = build(M, cls, C, xd, sd=seeded(cls, C, xd, seed=5, **kw), **kw)
    stacked = []
    if stack == "plain":
        a = build(M, "LoRACrossAttnProcessor", C, xd, rank=2, post_add=True,
                  sd=seeded("LoRACrossAttnProcessor", C, xd, seed=7, rank=2, post_add=True))
        b = build(M, "LoRACrossAttnProcessor", C, xd, rank=3, sd=seeded("LoRACrossAttnProcessor", C, xd, seed=8, rank=3))
        proc.inject_pre_lora(a)
        proc.inject_post_lora(b)
        stacked = [a, b]
    elif stack == "control":
        a = build(M, cls, C, xd, sd=seeded(cls, C, xd, seed=9, **kw), **kw)
        proc.inject_pre_lora(a)
        stacked = [a]
    g = torch.Generator().manual_seed(11)
    hs = torch.randn(2, 36, C, generator=g)
    ehs = torch.randn(2, 9, XD, generator=g) if cross else None
    w = torch.randn(2, 36, C, generator=g)
    h = hs.clone().requires_grad_(True)
    ctrls = []
    for p in [proc] + ([s for s in stacked if hasattr(s, "inject_control_states")] if stack == "control" else []):
        if hasattr(p, "inject_control_states"):
            cc = p.to_control.down.weight.shape[1] - (C if getattr(p, "concat_hidden", False) else 0)
            c = torch.randn(2, cc, 6, 6, generator=torch.Generator().manual_seed(13 + len(ctrls))).requires_grad_(True)
            p.inject_control_states(c)
            ctrls.append(c)
    y = proc(attn, h, ehs, None, scale)
    (y * w).sum().backward()
    grads = {n: summ(p.grad) for n, p in proc.named_parameters() if p.grad is not None}
    for i, s in enumerate(stacked):
        grads.update({f"stack{i}.{n}": summ(p.grad) for n, p in s.named_parameters() if p.grad is not None})
    return {"y": summ(y), "dh": summ(h.grad), "grads": grads, "dc": [summ(c.grad) for c in ctrls],
            "has_control": hasattr(proc, "inject_control_states")}


def run_unet(M, variant):
    """The training-step front half on a tiny SD-style UNet (the UNet restatement is the same for both modules): module M's
    ControlLoRA + processors with the wiring of train_text_to_image_control_lora.py:469-487."""
    from tests.check_unet import TINY, TINY_LORA

    torch.set_num_threads(1)
    kw = dict(TINY_LORA)
    kw.update({"v1": {}, "v2": dict(lora_control_version=2, lora_pre_conv_skipped=True), "post_add": dict(lora_post_add=True),
               "concat": dict(lora_concat_hidden=True, lora_control_rank=32, lora_pre_conv_skipped=True, lora_control_self_add=False)}[variant])
    cl = build(M, "ControlLoRA", sd=seeded("ControlLoRA", seed=0, **kw), **kw)
    u = UR.UNet2DConditionModel(**TINY)
    UR.init_synthetic_(u, seed=1)
    u.requires_grad_(False)
    MR.wire_processors(u, cl)
    g = torch.Generator().manual_seed(4)
    guide = torch.rand(2, 3, 128, 128, generator=g) * 2 - 1
    x = torch.randn(2, 4, 16, 16, generator=g)
    ehs = torch.randn(2, 77, TINY["cross_attention_dim"], generator=g)
    tgt = torch.randn(2, 4, 16, 16, generator=g)
    t = torch.tensor([10, 900])
    cl(guide)
    pred = u(x, t, ehs, cross_attention_kwargs={"scale": 0.8}).sample
    loss = torch.nn.functional.mse_loss(pred, tgt)
    loss.backward()
    return {"pred": summ(pred), "loss": float(loss), "grads": {n: summ(p.grad) for n, p in cl.named_parameters() if p.grad is not None}}


def main():
    from tests.golden import reference_import as RI

    R = RI.reference_models()
    gold = {"configs": {}, "hint": {}, "processor": {}, "unet": {}}
    for name in CONFIGS:
        cfg = RI.reference_config(name)
        gold["configs"][name] = cfg
        gold["hint"][name] = run_hint(R, cfg)
    for case in PROC_CASES:
        gold["processor"][case] = run_processor(R, case)
    for v in UNET_VARIANTS:
        gold["unet"][v] = run_unet(R, v)
    buf = []
    cases = pack(gold, buf)
    torch.save({"cases": cases, "flat": torch.tensor(buf, dtype=torch.float32)}, OUT)
    print("wrote", OUT, OUT.stat().st_size, "bytes")


if __name__ == "__main__":
    main()
