"""Inputs and seeded weights shared by tests/test_gpu_reference_live.py and oracle/gen_live_golden.py (which stores the
original project's outputs for them in tests/golden/live_cases.pt)."""
import torch

SAMPLE = 4096  # output elements kept per case


def randomize(module, seed, scale=None):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, prm in module.named_parameters():
            if prm.dim() == 1 and ("norm" in name or name.endswith(".0.weight")) and name.endswith("weight"):
                prm.copy_(1.0 + 0.1 * torch.randn(prm.shape, generator=g))
            elif prm.dim() == 1:
                prm.copy_(0.1 * torch.randn(prm.shape, generator=g))
            else:
                s = scale if scale is not None else prm.shape[-1] ** -0.5
                prm.copy_(s * torch.randn(prm.shape, generator=g))


def cross_attention_case():
    B, N, M, D, H = 2, 384, 2304, 1024, 8
    g = torch.Generator().manual_seed(2)
    x_q = torch.randn(1, N, D, generator=g)
    x_kv = torch.randn(B, M, D, generator=g) + 0.25
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[0, :333] = True
    pad[1, 2000:] = True
    return {"B": B, "N": N, "M": M, "D": D, "H": H, "xq": x_q.bfloat16(), "xkv": x_kv.bfloat16(), "pad": pad}


def encoder_kwargs():
    B, M, C, N, D = 2, 3000, 256, 320, 512
    kw = dict(C=C, num_latents=N, num_latent_channels=D, num_cross_attention_heads=4, num_cross_attention_layers=2,
              first_cross_attention_layer_shared=False, num_self_attention_heads=8, num_self_attention_layers_per_block=2,
              num_self_attention_blocks=2, first_self_attention_block_shared=True, num_cross_attention_qk_channels=256,
              num_cross_attention_v_channels=512)
    g = torch.Generator().manual_seed(6)
    x = (torch.randn(B, M, C, generator=g) + 0.1).bfloat16()
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[1, 2500:] = True
    return kw, (x, pad)


def csm_config():
    cfg = dict(vocab_size=262, max_seq_len=1536, max_latents=512, num_channels=512, num_heads=8, num_self_attention_layers=3,
               num_self_attention_rotary_layers=1, cross_attention_dropout=0.0, output_norm=True, abs_pos_emb=False,
               init_scale=0.05)
    g = torch.Generator().manual_seed(8)
    B, n0, prefix = 2, 1400, 1000
    tokens = torch.randint(0, 262, (B, n0 + 3), generator=g)
    pad = torch.zeros(B, n0 + 3, dtype=torch.bool)
    pad[1, :57] = True
    return cfg, (tokens, pad, n0, prefix)


def grad_case():
    cfg = dict(vocab_size=64, max_seq_len=192, max_latents=64, num_channels=128, num_heads=4, num_self_attention_layers=2,
               num_self_attention_rotary_layers=1, cross_attention_dropout=0.0, output_norm=True, abs_pos_emb=False,
               init_scale=0.05)
    g = torch.Generator().manual_seed(12)
    tokens = torch.randint(0, 64, (2, 160), generator=g)
    pad = torch.zeros(2, 160, dtype=torch.bool)
    pad[1, :9] = True
    target = torch.randint(0, 64, (2, 64), generator=g)
    names = ["cross_attention.0.module.attention.q_proj.weight", "cross_attention.0.module.attention.k_proj.weight",
             "self_attention.0.0.module.attention.q_proj.weight", "self_attention.0.0.module.attention.k_proj.weight",
             "self_attention.1.0.module.attention.v_proj.weight"]
    return cfg, (tokens, pad, target, names)
