"""Two Sigma-tiny training steps (forward with labels, backward, AdamW) under torch.use_deterministic_algorithms(True), from fixed
seeds, saving the losses, every gradient and every updated parameter to --out.  Two runs of this script must save bitwise-equal
tensors (tests/test_deterministic_gpu.py).  Needs CUBLAS_WORKSPACE_CONFIG=:4096:8 in the environment, as torch requires for
cuBLAS under the switch; torch's NaN fill of uninitialised memory stays on.

    CUBLAS_WORKSPACE_CONFIG=:4096:8 python scripts/det_train_steps.py --amp {fp32,bf16} --out run.pt [--height 72 --width 104]
"""
import argparse
import contextlib
import io
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--amp", default="fp32", choices=["fp32", "bf16"])
    ap.add_argument("--out", required=True)
    ap.add_argument("--height", type=int, default=72)
    ap.add_argument("--width", type=int, default=104)
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--classes", type=int, default=9)
    a = ap.parse_args()
    from sigma_b200 import modules as M, train_util
    torch.use_deterministic_algorithms(True)
    assert torch.utils.deterministic.fill_uninitialized_memory
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    torch.manual_seed(0)
    cfg = types.SimpleNamespace(backbone="sigma_tiny", decoder="MambaDecoder", num_classes=a.classes, image_height=a.height,
                                image_width=a.width, pretrained_model=None, bn_eps=1e-3, bn_momentum=0.1)
    with contextlib.redirect_stdout(io.StringIO()):
        model = M.EncoderDecoder(cfg, criterion=torch.nn.CrossEntropyLoss(reduction="mean", ignore_index=255)).cuda().train()
    opt = train_util.make_optimizer(model)
    step = train_util.TrainStep(model, opt, amp_dtype=torch.bfloat16 if a.amp == "bf16" else None)
    g = torch.Generator().manual_seed(1234)
    out = {}
    for i in range(2):
        rgb = torch.randn(a.batch, 3, a.height, a.width, generator=g).cuda()
        mx = torch.randn(a.batch, 3, a.height, a.width, generator=g).cuda()
        gt = torch.randint(0, a.classes, (a.batch, a.height, a.width), generator=g).cuda()
        gt[:, : a.height // 8] = 255                                   # ignored pixels
        out[f"loss{i}"] = step(rgb, mx, gt).detach().float().cpu()
    for n, p in model.named_parameters():
        out["param." + n] = p.detach().cpu()
        if p.grad is not None:
            out["grad." + n] = p.grad.detach().cpu()
    for n, b in model.named_buffers():
        out["buffer." + n] = b.detach().cpu()
    torch.save(out, a.out)
    print(f"saved {len(out)} tensors, losses {float(out['loss0']):.6f} {float(out['loss1']):.6f}")


if __name__ == "__main__":
    main()
