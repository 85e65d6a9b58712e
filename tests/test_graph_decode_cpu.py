"""CPU checks of the graph decoder's host rules: the key windows against the 🤗 wrapper's truncation loop restated with
real tensors, the in-graph position rule against ``positions()``, and the refusals that need no GPU."""
import pytest
import torch


def _truncation_loop(prompt_len, prefix_len, steps, max_seq_len, max_latents):
    """The cache lengths of a one-token generation loop, truncated as the 🤗 wrapper truncates (the loop of the FP8
    KV-cache generation test), tracked as the token indices the caches hold."""
    ca = list(range(prompt_len))
    sa = list(range(prefix_len, prompt_len))
    out = []
    for s in range(steps):
        tok = prompt_len + s
        n = len(ca) + 1
        if n > max_seq_len:
            ca = ca[n - max_seq_len:]
            n = max_seq_len
        nlat = len(sa) + 1
        if nlat > max_latents:
            sa = sa[nlat - max_latents:]
            nlat = max_latents
        ca, sa = ca + [tok], sa + [tok]
        out.append((ca[0], ca[-1] + 1, sa[0] - prefix_len, sa[-1] + 1 - prefix_len, n - nlat))
        assert len(ca) == n and len(sa) == nlat and ca[-nlat:] == sa
    return out


@pytest.mark.parametrize("prompt_len,prefix_len,steps,max_seq_len,max_latents", [
    (20, 0, 30, 64, 48),      # prompt shorter than max_latents, no prefix: the latents fill, then the prefix grows
    (48, 0, 10, 64, 48),      # prompt equal to max_latents
    (120, 90, 60, 160, 48),   # longer: both windows slide (the GPU test's geometry)
    (100, 30, 50, 110, 48),   # a prompt whose latents overflow at the first step
    (160, 112, 5, 160, 48),   # a full context: the cross-attention window slides from the first step
    (5, 4, 3, 8, 2),
])
def test_windows_follow_the_truncation_loop(prompt_len, prefix_len, steps, max_seq_len, max_latents):
    from perceiver_io_b200 import decode_windows

    got = [tuple(w) for w in decode_windows(prompt_len, prefix_len, steps, max_seq_len, max_latents)]
    assert got == _truncation_loop(prompt_len, prefix_len, steps, max_seq_len, max_latents)


def test_position_rule_matches_positions_with_left_padding():
    from perceiver_io_b200 import positions
    from perceiver_io_b200.generation import decode_windows, window_positions

    B, n0, prefix, steps, cap = 3, 30, 12, 25, 60
    pad = torch.zeros(B, cap, dtype=torch.uint8)
    pad[1, :4] = 1
    pad[2, :n0] = 1                      # a fully padded prompt row
    cols = torch.arange(cap, dtype=torch.int32)
    for w in decode_windows(n0, prefix, steps, 40, 16):
        window = torch.tensor([w.ca_begin, w.ca_end], dtype=torch.int32)
        n = w.ca_end - w.ca_begin
        shift = pad[:, w.ca_begin:w.ca_end].bool().sum(dim=1, keepdim=True)
        want = positions(B, n, shift=shift)[:, -1:]
        assert torch.equal(window_positions(pad, window, cols), want)


def _small_model():
    import perceiver_io_b200 as P

    cfg = P.CausalSequenceModelConfig(vocab_size=97, max_seq_len=160, max_latents=48, num_channels=128, num_heads=4,
                                      num_self_attention_layers=2, cross_attention_dropout=0.0)
    return P.CausalSequenceModel(cfg)


def test_refusals_without_a_gpu():
    from perceiver_io_b200 import GraphedDecoder

    model = _small_model().eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        GraphedDecoder(model, batch=2, max_new_tokens=8)
    with pytest.raises(RuntimeError, match="eval mode"):
        GraphedDecoder(model.train(), batch=2, max_new_tokens=8)
    with pytest.raises(ValueError, match="max_new_tokens"):
        GraphedDecoder(model.eval(), batch=2, max_new_tokens=0)
    with pytest.raises(ValueError, match="kv_cache"):
        GraphedDecoder(model, batch=2, max_new_tokens=4, kv_cache="int8")
    with pytest.raises(TypeError, match="CausalSequenceModel"):
        GraphedDecoder(model.self_attention, batch=2, max_new_tokens=4)
