"""Runs the parity checkers (tests/check_*.py) in host-logic mode: CLB_EMU=1, every kernel wrapper replaced by its torch
restatement (tests/emu_ops.py), everything above the C ABI - tape engine, LoRA slot packing, control algebra, hint-encoder
program, Trainer - is the product code and is compared with the fp32 oracle exactly as the `-m gpu` suite does on an H100.

usage: python tests/run_emulated.py [case ...]      (prints one `RESULT <case> OK|FAIL <seconds>` line per case)
Must be its own process: the mode is chosen when the first checker is imported (tests/_device.py)."""
import contextlib
import io
import os
import sys
import time
import traceback
from pathlib import Path

os.environ["CLB_EMU"] = "1"
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def _cases():
    from tests import check_clip, check_hint, check_unet, check_vae

    c = {}
    for v in ("none", "plain", "v1", "v2", "v1_stacked", "v1_post_add", "v1_concat", "v1_stacked@0.5", "v2@0.5", "v1_stacked@0.0"):
        c["unet_" + v] = lambda v=v: check_unet.run(v)
    for k in ("hint_v1", "hint_v2", "train_v1", "train_v2", "train_lora_only", "resume", "accumulate"):
        c[k] = check_hint.CASES[k]
    c["vae_tiny"] = lambda: check_vae.run("tiny")
    c["clip_tiny"] = lambda: check_clip.run("tiny")
    from tests import check_eager, check_reference_golden, check_sampler, check_variants

    c.update(check_variants.CASES)
    c.update(check_eager.CASES)
    c.update(check_reference_golden.CASES)
    c.update(check_sampler.CASES)
    return c


def main():
    import torch

    torch.set_num_threads(min(8, os.cpu_count() or 1))
    cases = _cases()
    names = sys.argv[1:] or list(cases)
    bad = 0
    for n in names:
        t0 = time.time()
        buf = io.StringIO()
        try:
            with contextlib.redirect_stdout(buf):
                ok = bool(cases[n]())
        except Exception:
            ok = False
            buf.write(traceback.format_exc())
        if not ok:
            bad += 1
            print(buf.getvalue(), flush=True)
        print(f"RESULT {n} {'OK' if ok else 'FAIL'} {time.time() - t0:.1f}", flush=True)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
