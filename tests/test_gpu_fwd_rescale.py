"""-m gpu: the forward kernel rescales the running numerator O only when a row maximum moved in a warp.

After the first key tile, a warp skips the rescale of O when no row of its 16 moved its maximum.  Here exactly one row
of every warp takes its maximum in a later key tile (the key tile, 2 to 6, and the row position vary with the warp), and every other row
keeps the maximum it found in key 0.  So in one key tile some warps rescale and others skip, and inside a rescaling
warp most rows have alpha = 1.  A skipped rescale of a moved row is off by about e^-4, far outside the fp64 gate.

The call runs on the whole-unit plan (N > 66 * 128 on a 132-SM H100), where one segment covers every key tile, so
the late key tiles go through the pipelined steady-state loop."""
import pytest
import torch

from fwd_variants import case_id, plan_segments, workers_for
from gpu_util import assert_parity

pytestmark = pytest.mark.gpu

DTYPE = {"bf16": torch.bfloat16, "fp16": torch.float16}
B, H, N, M, DV = 1, 1, 8600, 1000, 128   # M: 8 key tiles, the last one ragged (masked path)


LATE = 5  # late keys, one per key tile 2..6


def _operands(dqk, dtype):
    """Scores ~ N(0, 1) except: key 0 scores ~8 against every row; late key c (in key tile 2 + c) scores ~4 against
    every row but the special rows of class c, against which it scores ~12.  Warp group g (rows 16 g .. 16 g + 15) has
    one special row, 16 g + (5 g mod 16), of class g mod 5."""
    g = torch.Generator(device="cuda").manual_seed(5)
    basis = torch.linalg.qr(torch.randn(dqk, 1 + LATE, generator=g, device="cuda"))[0]
    u, w = basis[:, 0], basis[:, 1:].T
    q = dqk ** 0.5 * u + 0.25 * torch.randn(N, dqk, generator=g, device="cuda")
    k = torch.randn(M, dqk, generator=g, device="cuda")
    v = torch.randn(M, DV, generator=g, device="cuda")
    k[0] = 8.0 * u
    late = [128 * (2 + c) + 37 for c in range(LATE)]
    for c in range(LATE):
        k[late[c]] = 4.0 * u + 8.0 * w[c]
    grp = torch.arange(N // 16, device="cuda")
    rows = 16 * grp + (5 * grp) % 16
    q[rows] += dqk ** 0.5 * w[grp % LATE]
    keys = torch.tensor(late, device="cuda")[grp % LATE]
    return q[None].to(dtype), k[None].to(dtype), v[None].to(dtype), rows, keys


@pytest.mark.parametrize("pair", [False, True], ids=["single", "pair"])
@pytest.mark.parametrize("dqk", [64, 128])
@pytest.mark.parametrize("dt", list(DTYPE))
def test_rescale_only_moved_rows(dt, dqk, pair):
    from perceiver_io_b200 import ops

    name = case_id((dqk, DV, dt, pair))
    counts, _ = plan_segments(B, H, N, M, workers_for(ops.device_info()["num_sms"], pair), pair)
    assert counts["slots"] == 0, "expected the whole-unit plan"
    q, k, v, rows, keys = _operands(dqk, DTYPE[dt])
    scale = dqk ** -0.5

    # the construction: the special rows peak at their late key, every other row at key 0
    arg = (q[0].double() @ k[0].double().T).argmax(-1)
    special = torch.zeros(N, dtype=torch.bool, device="cuda")
    special[rows] = True
    assert torch.equal(arg[rows], keys), f"{name}: a special row does not peak at its late key"
    assert (arg[~special] == 0).all(), f"{name}: a row other than the special ones does not peak at key 0"

    out = ops.attention(q, k, v, H, scale, impl="tcgen05_pair" if pair else "tcgen05")
    assert_parity(out, q, k, v, H, scale, what=f"{name} late maxima", per_row=True)
