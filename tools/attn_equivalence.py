"""Equivalence check of the attention ops between two builds of the package (e.g. before and after a host-side
refactor): the same seeded calls, run once per build in separate processes, saved, then compared.

    python tools/attn_equivalence.py run --root <tree of build A> --out a1.pt     # at least twice for the reference
    python tools/attn_equivalence.py run --root <tree of build A> --out a2.pt     # build, to learn its run-to-run spread
    python tools/attn_equivalence.py run --root <tree of build B> --out b1.pt
    python tools/attn_equivalence.py compare --ref a1.pt a2.pt --new b1.pt

Every call records its results (tensors, booleans, or the type and text of the error it raised) and how far
``_lib.launch_count()`` advanced.  ``compare`` requires equal launch counts, equal booleans and errors, and tensors of
B bitwise equal to A wherever A's runs agree bitwise.  grad_q accumulated with fp32 atomics (head dims up to 128) is
held to A's own run-to-run difference instead, and to at least one rounding step of its dtype.  Needs a GPU."""
from __future__ import annotations

import argparse
import sys

import torch

# head dims reaching every backward box pair (NQB, NVB) in {1, 2, 3}^2
SHAPES = [(64, 64), (128, 128), (131, 131), (32, 160), (64, 128), (128, 64), (160, 64), (184, 120), (120, 184)]
# (operand dtype, batch-1 q, pad mask, causal)
VARIANTS = [(torch.bfloat16, True, True, False), (torch.float32, False, False, True), (torch.bfloat16, False, True, True),
            (torch.float16, True, False, True)]
B, N, M, H, SEED = 2, 200, 700, 2, 0x5EED


def _inputs(dqk, dv, dtype, bq1, with_pad, g):
    q = torch.randn(1 if bq1 else B, N, H * dqk, generator=g)
    k = torch.randn(B, M, H * dqk, generator=g)
    v = torch.randn(B, M, H * dv, generator=g)
    go = torch.randn(B, N, H * dv, generator=g)
    pad = None
    if with_pad:
        pad = torch.zeros(B, M, dtype=torch.bool)
        pad[0, 650:] = True
        pad[1, 301:] = True
    to = lambda t: None if t is None else t.cuda()
    return [to(t.to(dtype)) for t in (q, k, v, go)] + [to(pad)]


def run(root: str, out_path: str) -> None:
    sys.path.insert(0, root)
    from perceiver_io_b200 import _lib, ops

    results = {}

    def record(name, fn, atomic=()):
        torch.cuda.synchronize()
        before = _lib.launch_count()
        try:
            r = fn()
            r = r if isinstance(r, (tuple, list)) else (r,)
            value = [t.detach().cpu().clone() if torch.is_tensor(t) else t for t in r]
        except Exception as e:  # noqa: BLE001 - the error itself is a result to compare
            value = f"{type(e).__name__}: {e}"
        torch.cuda.synchronize()
        results[name] = {"launches": _lib.launch_count() - before, "value": value, "atomic": list(atomic)}

    g = torch.Generator().manual_seed(SEED)
    for dqk, dv in SHAPES:
        for dtype, bq1, with_pad, causal in VARIANTS:
            q, k, v, go, pad = _inputs(dqk, dv, dtype, bq1, with_pad, g)
            scale = dqk ** -0.5
            atomic_dq = max(dqk, dv) <= 128  # grad_q is accumulated with fp32 atomics up to head dim 128 (padded)
            tag = f"{dqk}/{dv} {str(dtype)[6:]} bq1={bq1} pad={with_pad} causal={causal}"
            kw = dict(pad_mask=pad, causal=causal)
            record(f"{tag} attention", lambda: ops.attention(q, k, v, H, scale, **kw))
            record(f"{tag} tcgen05_supported", lambda: ops.tcgen05_supported(q, k, v, H, **kw))
            for p in (0.0, 0.1):
                def autograd(p=p):
                    leaves = [t.detach().clone().requires_grad_() for t in (q, k, v)]
                    o = ops.attention(*leaves, H, scale, dropout_p=p, dropout_seed=77, **kw)
                    o.backward(go.to(o.dtype))
                    return [o] + [t.grad for t in leaves]
                record(f"{tag} attention autograd p={p}", autograd, atomic=(1,) if atomic_dq else ())

            m0 = 256  # a key shard [256, 700) of the 700 keys
            ks, vs, pads = k[:, m0:], v[:, m0:], None if pad is None else pad[:, m0:]
            for p in (0.0, 0.1):
                record(f"{tag} attention_partial p={p}",
                       lambda p=p: ops.attention_partial(q, k, v, H, scale, dropout_p=p, dropout_seed=5, **kw))
                record(f"{tag} attention_partial shard p={p}",
                       lambda p=p: ops.attention_partial(q, ks, vs, H, scale, pad_mask=pads, causal=causal, m_total=M,
                                                         m_offset=m0, dropout_p=p, dropout_seed=5))

            po, pm, pl = ops.attention_partial(q, k, v, H, scale, **kw)
            out = ops.combine_partials(po[None], pm[None], pl[None], ops._compute_dtype(dtype))
            for p in (0.0, 0.1):
                bw = dict(pad_mask=pad, causal=causal, dropout_p=p, dropout_seed=9)
                record(f"{tag} attention_backward check p={p}",
                       lambda bw=bw: ops.attention_backward(q, k, v, out, go, pm, pl, H, scale, check_only=True, **bw))
                record(f"{tag} attention_backward p={p}",
                       lambda bw=bw: ops.attention_backward(q, k, v, out, go, pm, pl, H, scale, **bw),
                       atomic=(0,) if atomic_dq else ())
                sw = dict(pad_mask=pads, causal=causal, dropout_p=p, dropout_seed=9)
                record(f"{tag} attention_backward_shard check p={p}",
                       lambda sw=sw: ops.attention_backward_shard(q, ks, vs, out, go, pm, pl, H, scale, M, m0,
                                                                  check_only=True, **sw))
                record(f"{tag} attention_backward_shard p={p}",
                       lambda sw=sw: ops.attention_backward_shard(q, ks, vs, out, go, pm, pl, H, scale, M, m0, **sw),
                       atomic=(0,) if atomic_dq else ())
            record(f"{tag} attention_dropout_forward",
                   lambda: ops.attention_dropout_forward(q, k, v, pm, pl, H, scale, 0.1, 11, **kw))

            if dqk % 16 == 0 and dv % 16 == 0:
                qd, kd = (t.float().reshape(*t.shape[:2], H, -1).abs().amax(dim=(0, 1, 3)) / 448 for t in (q, k))
                vd = v.float().reshape(B, M, H, dv).abs().amax(dim=(0, 1)) / 448
                q8, k8 = ops.fp8_quantize(q, qd, H), ops.fp8_quantize(k, kd, H)
                vt8 = ops.fp8_transpose_v(ops.fp8_quantize(v, vd, H), H)
                for partial in (False, True):
                    record(f"{tag} attention_fp8 partial={partial}",
                           lambda partial=partial: ops.attention_fp8(q8, k8, vt8, qd, kd, vd, H, scale, partial=partial,
                                                                     **kw))
    _modules(record)
    torch.save(results, out_path)
    print(f"{len(results)} calls -> {out_path}")


def _modules(record):
    """The modules' routing (modules.py): seeded module calls recording the output, the parameter and input gradients
    of autograd calls (held as fp32-atomics results: they sit downstream of grad_q), the returned caches and their
    dtypes, and, as the fingerprint of the routes taken, the ``_pcv_*`` slots each module holds afterwards."""
    import perceiver_io_b200 as P
    from perceiver_io_b200 import modules

    dev = "cuda"

    def fresh(model):
        for m in model.modules():
            for k in [k for k in m.__dict__ if k.startswith("_pcv_")]:
                del m.__dict__[k]
        return model

    def slots(model):
        return sorted(f"{n}.{k}" for n, m in model.named_modules() for k in m.__dict__ if k.startswith("_pcv_"))

    def call(name, model, inputs, grad=False, seed=0, autocast=False):
        def fn():
            fresh(model).zero_grad(set_to_none=True)
            ins = [t.detach().clone().requires_grad_(grad) for t in inputs]
            torch.manual_seed(seed)
            with torch.set_grad_enabled(grad), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                out = model(*ins).last_hidden_state
            if not grad:
                return [out, slots(model)]
            out.float().square().sum().backward()
            grads = [p.grad for _, p in sorted(model.named_parameters())] + [t.grad for t in ins]
            return [out, slots(model)] + grads
        n_grads = len(list(model.parameters())) + len(inputs) if grad else 0
        record(f"modules {name}", fn, atomic=tuple(range(2, 2 + n_grads)))

    def cross(dtype, dropout=0.0):
        torch.manual_seed(1)
        return P.CrossAttention(num_heads=4, num_q_input_channels=256, num_kv_input_channels=512,
                                dropout=dropout).to(dev, dtype)

    g = torch.Generator().manual_seed(SEED + 1)
    x_q = torch.randn(1, 256, 256, generator=g).to(dev)
    for M in (256, 1024):
        x_kv = torch.randn(2, M, 512, generator=g).to(dev)
        for dtype in (torch.bfloat16, torch.float32):
            call(f"CrossAttention eval M={M} {str(dtype)[6:]}", cross(dtype).eval(), [x_q.to(dtype), x_kv.to(dtype)])
        call(f"CrossAttention eval M={M} autocast", cross(torch.float32).eval(), [x_q, x_kv], autocast=True)
        modules.fp8_config["enabled"] = True
        try:
            call(f"CrossAttention eval M={M} fp8", cross(torch.bfloat16).eval(), [x_q.bfloat16(), x_kv.bfloat16()])
        finally:
            modules.fp8_config["enabled"] = False
    x_kv = x_kv.bfloat16()
    for training in (False, True):
        for p in (0.0, 0.1):
            modules.kv_producer_config["training"] = training
            try:
                call(f"CrossAttention train route={training} p={p}", cross(torch.bfloat16, p).train(),
                     [x_q.bfloat16(), x_kv], grad=True, seed=3)
            finally:
                modules.kv_producer_config["training"] = False

    for n in (128, 512, 2048):  # 256, 1024 and 4096 latent rows: below min_rows, the eager band, min_rows_latent
        torch.manual_seed(2)
        sa = P.SelfAttention(num_heads=4, num_channels=256).to(dev, torch.bfloat16)
        x = torch.randn(2, n, 256, generator=g).to(dev, torch.bfloat16)
        call(f"SelfAttention eval rows={2 * n}", sa.eval(), [x])
        for training in (False, True):
            modules.kv_producer_config["training"] = training
            try:
                call(f"SelfAttention train rows={2 * n} route={training}", sa.train(), [x], grad=True)
            finally:
                modules.kv_producer_config["training"] = False

    torch.manual_seed(4)
    cfg = P.CausalSequenceModelConfig(vocab_size=64, max_seq_len=96, max_latents=32, num_channels=128, num_heads=4,
                                      num_self_attention_layers=2, cross_attention_dropout=0.0)
    model = P.CausalSequenceModel(cfg).to(dev, torch.bfloat16).eval()
    tokens = torch.randint(0, 64, (2, 64 + 16), generator=g).to(dev)

    def generate():
        fresh(model)
        with torch.no_grad():
            out = model(tokens[:, :64], prefix_len=32, kv_cache=[])
            logits, cache, pos = [out.logits], out.kv_cache, 64
            for step in range(8):
                m = 5 if step == 3 else 1
                if step == 5:  # beam reordering
                    cache = [(k.index_select(0, torch.tensor([1, 0], device=dev)),
                              v.index_select(0, torch.tensor([1, 0], device=dev))) for k, v in cache]
                out = model(tokens[:, pos:pos + m], prefix_len=32, kv_cache=cache)
                logits.append(out.logits)
                cache, pos = out.kv_cache, pos + m
        return logits + [t for kv in cache for t in kv] + [[str(k.dtype) for k, _ in cache], slots(model)]

    for kv8 in (False, True):
        modules.fp8_config["kv_cache"] = kv8
        try:
            record(f"modules CausalSequenceModel decode kv8={kv8}", generate)
        finally:
            modules.fp8_config["kv_cache"] = False


def _same(a, b):
    """Bitwise equality (NaNs included) of two tensors of one dtype and shape."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    bits = lambda t: t.contiguous().view(torch.uint8) if t.dtype.is_floating_point else t
    return torch.equal(bits(a), bits(b))


def compare(ref_paths, new_paths) -> int:
    refs = [torch.load(p) for p in ref_paths]
    news = [torch.load(p) for p in new_paths]
    bad, bitwise, held = [], 0, []
    names = set(refs[0])
    if any(set(r) != names for r in refs + news):
        bad.append("the runs made different calls")
    for name in sorted(names.intersection(*map(set, refs + news))):
        launches = {r[name]["launches"] for r in refs + news}
        if len(launches) != 1:
            bad.append(f"{name}: launches {[r[name]['launches'] for r in refs]} -> {[r[name]['launches'] for r in news]}")
        rv, nv = [r[name]["value"] for r in refs], [r[name]["value"] for r in news]
        if any(isinstance(v, str) for v in rv + nv):  # an error in some run
            if not all(isinstance(v, str) and v == rv[0] for v in rv + nv):
                bad.append(f"{name}: {rv[0]!r} -> {nv[0]!r}")
            continue
        if any(len(v) != len(rv[0]) for v in rv + nv):
            bad.append(f"{name}: the number of results differs")
            continue
        for i, x in enumerate(rv[0]):
            if not torch.is_tensor(x):
                if any(v[i] != x for v in rv + nv):
                    bad.append(f"{name}[{i}]: {x!r} -> {[v[i] for v in nv]!r}")
                continue
            if all(_same(x, v[i]) for v in rv[1:] + nv):
                bitwise += 1
                continue
            if any(v[i].shape != x.shape or v[i].dtype != x.dtype for v in nv):
                bad.append(f"{name}[{i}]: shape or dtype changed")
                continue
            dist = lambda a, b: (a.double() - b.double()).abs().max().item()
            ref_spread = max(dist(a[i], b[i]) for j, a in enumerate(rv) for b in rv[j + 1:])
            diff = max(dist(x, v[i]) for v in nv)
            atomic = i in refs[0][name]["atomic"]
            # the order of fp32 atomics is random: when the reference runs happen to agree, one rounding step of the
            # output at its largest magnitude is the least a different order can move it
            bound = max(ref_spread, torch.finfo(x.dtype).eps * x.abs().max().item()) if atomic else ref_spread
            held.append(f"{name}[{i}]{' (fp32 atomics)' if atomic else ''}: reference run-to-run {ref_spread:.3e}, "
                        f"new vs reference {diff:.3e}, bound {bound:.3e}")
            if diff > bound:
                bad.append(held[-1])
    print(f"{len(names)} calls, {len(refs)} reference and {len(news)} new runs: {bitwise} tensors bitwise equal in every "
          f"run, {len(held)} held to a bound, {len(bad)} mismatches")
    for line in held:
        print("  held: " + line)
    for line in bad:
        print("  MISMATCH: " + line)
    return 1 if bad else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="cmd", required=True)
    r = sub.add_parser("run")
    r.add_argument("--root", required=True, help="directory holding the perceiver_io_b200 package to test")
    r.add_argument("--out", required=True)
    c = sub.add_parser("compare")
    c.add_argument("--ref", nargs="+", required=True, help="results of the reference build, two runs or more")
    c.add_argument("--new", nargs="+", required=True, help="results of the build under test")
    args = ap.parse_args()
    if args.cmd == "run":
        run(args.root, args.out)
    else:
        sys.exit(compare(args.ref, args.new))
