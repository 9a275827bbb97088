"""Diagnostic: gradients with weight gradients on the side stream vs on the main stream (development aid)."""
import os, sys, copy
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE); sys.path.insert(0, os.path.join(HERE, "..")); sys.path.insert(0, os.path.join(HERE, "..", "ml-mdm_b200"))
import torch
import parity
import tiny_configs as tc

def grads(kind, steps=3):
    model, _, _ = parity.tiny_model(tc.TINY[kind])
    model = model.cuda()
    nlev = 1 if kind == "unet" else 2
    out = []
    for s in range(steps):
        x, t, lm, mask = tc.seeded_inputs(5, 2, 16 if nlev == 1 else 32, 6, nlevels=nlev)
        xs = x.cuda() if nlev == 1 else [xi.cuda() for xi in x]
        o = model(xs, t.cuda(), lm.cuda(), mask.cuda(), {})
        os_ = list(o) if isinstance(o, list) else [o]
        sum((a * a).sum() for a in os_).backward()
        torch.cuda.synchronize()
        out.append({k: p.grad.detach().clone() for k, p in model.named_parameters()})
        model.zero_grad(set_to_none=True)
    return out

if __name__ == "__main__":
    kind = sys.argv[1] if len(sys.argv) > 1 else "unet"
    g = grads(kind)
    torch.save(g, f"/tmp/diag_{kind}_{os.environ.get('MDM_SIDE_WGRAD','auto')}_{os.environ.get('MDM_NO_GRAPH','g')}.pt")
    ref_path = sys.argv[2] if len(sys.argv) > 2 else None
    if ref_path:
        ref = torch.load(ref_path)
        for s, (a, b) in enumerate(zip(g, ref)):
            bad = []
            for k in a:
                nb = float(b[k].norm()); na = float(a[k].norm())
                e = float((a[k] - b[k]).norm()) / max(nb, 1e-30)
                if e > 5e-2:
                    bad.append((k, round(na / max(nb, 1e-30), 3), round(e, 3)))
            print(f"step {s}: {len(bad)} mismatching of {len(a)}:", bad[:12])
