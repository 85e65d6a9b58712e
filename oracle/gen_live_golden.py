"""Stored yardsticks for tests/test_gpu_reference_live.py: runs the ORIGINAL project (krasserm/perceiver-io, importable
from baseline/_ref after `python baseline/install_ref.py`) on the CPU and writes tests/golden/live_cases.pt.

Per case: a fixed, seeded sample of the fp64 reference output (indices + values), max|eager bf16 - fp64| over the
WHOLE output (the eager arm is the reference's own code in bf16: .bfloat16() or CPU autocast), and max|fp64|, so the
GPU test can apply the derived gate  max|ours - ref64| <= 2 * eager_err + 1e-3 * max|ref64|  on the sample.  The model
weights are not stored: the test builds the package's modules, whose parameter names and shapes match the reference's,
and draws the same seeded weights.

    python oracle/gen_live_golden.py        (needs baseline/_ref; CPU only)
"""
import copy
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "baseline"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import install_ref  # noqa: E402
from live_cases import SAMPLE, cross_attention_case, csm_config, encoder_kwargs, grad_case, randomize  # noqa: E402

core = install_ref.import_reference_core()


class PassThrough(core.InputAdapter):
    def forward(self, x):
        return x


def pack(ref64, eager, seed):
    flat = ref64.reshape(-1)
    g = torch.Generator().manual_seed(seed)
    idx = torch.randperm(flat.numel(), generator=g)[:SAMPLE].clone()
    return {"idx": idx, "ref": flat[idx].clone(), "eager_err": (eager.double() - ref64).abs().max().item(),
            "ref_max": ref64.abs().max().item()}


@torch.no_grad()
def main():
    torch.set_num_threads(os.cpu_count() or 1)
    out = {}
    # (1) CrossAttention, north-star head geometry
    a = cross_attention_case()
    ref = core.CrossAttention(num_heads=a["H"], num_q_input_channels=a["D"], num_kv_input_channels=a["D"]).eval()
    randomize(ref, 1)
    ref.attention.q_proj.weight.mul_(3.0)
    r64 = copy.deepcopy(ref).double()(a["xq"].double(), a["xkv"].double(), pad_mask=a["pad"]).last_hidden_state
    eager = copy.deepcopy(ref).bfloat16()(a["xq"], a["xkv"], pad_mask=a["pad"]).last_hidden_state
    cpu = ref(a["xq"].float(), a["xkv"].float(), pad_mask=a["pad"]).last_hidden_state
    out["cross"] = pack(r64, eager, 1)
    out["cross_cpu32"] = pack(cpu.double(), eager, 1)
    # (2) PerceiverEncoder
    kw, (x, pad) = encoder_kwargs()
    enc = core.PerceiverEncoder(PassThrough(kw.pop("C")), **kw).eval()
    randomize(enc, 5)
    r64 = copy.deepcopy(enc).double()(x.double(), pad_mask=pad)
    eager = copy.deepcopy(enc).bfloat16()(x, pad_mask=pad)
    out["encoder"] = pack(r64, eager, 2)
    # (3) Perceiver AR: full forward logits and the uncached logits of the 3 decode positions
    m = core.CausalSequenceModel(core.CausalSequenceModelConfig(**csm_config()[0])).eval()
    randomize(m, 7, scale=0.04)
    t, p, n0, prefix = csm_config()[1]
    m64 = copy.deepcopy(m).double()
    r64 = m64(t[:, :n0], prefix_len=prefix, pad_mask=p[:, :n0]).logits
    r64_all = m64(t, prefix_len=prefix, pad_mask=p).logits
    with torch.autocast("cpu", dtype=torch.bfloat16):
        eager = m(t[:, :n0], prefix_len=prefix, pad_mask=p[:, :n0]).logits
        eager_all = m(t, prefix_len=prefix, pad_mask=p).logits
    out["csm_full"] = pack(r64, eager, 3)
    for s in range(3):
        j = n0 - prefix + s
        out[f"csm_step{s}"] = pack(r64_all[:, j], eager_all[:, j], 4 + s)
    # (4) gradients of q/k/v projections through rotary: the reference's fp32 autograd
    cfg, (tokens, pad, target, names) = grad_case()
    ref = core.CausalSequenceModel(core.CausalSequenceModelConfig(**cfg))
    randomize(ref, 11, scale=0.06)
    ref.train()
    with torch.enable_grad():
        logits = ref(tokens, prefix_len=96, pad_mask=pad).logits
        torch.nn.functional.cross_entropy(logits.reshape(-1, 64), target.reshape(-1)).backward()
    prm = dict(ref.named_parameters())
    out["grads"] = {n: prm[n].grad.detach().float().clone() for n in names}
    path = os.path.join(ROOT, "tests", "golden", "live_cases.pt")
    torch.save(out, path)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
