"""CPU estimate for the bridge fields (SPATIALSIRENAUGDISENTANGLE, RESSIRENDISENTANGLE): fp16 wgmma operands in the trunk,
the 3-wide bridge head and the colour branch, against float64.  Init distributions as in the reference
(siren.py:904-1082): frequency_init(25) where the reference applies it, nn.Linear's default elsewhere.  RES is also run with
its density chain scaled so that max |a| = 1 and c = 0 (a . v is then O(1)), which is how the tests exercise the
density-from-v path; its sigma error is v's error times |a|.

    python tools/bridge_precision.py"""
import math
import torch

D = torch.float64
N = 20000
H = 256


def lin(fan_in, fan_out, kind):
    w = torch.empty(fan_out, fan_in, dtype=D)
    bb = 1 / math.sqrt(fan_in)
    if kind == "first":
        w.uniform_(-1 / fan_in, 1 / fan_in)
    elif kind == "freq":
        b = math.sqrt(6 / fan_in) / 25
        w.uniform_(-b, b)
    else:  # nn.Linear default: kaiming_uniform(a=sqrt 5) -> U(+-1/sqrt(fan_in))
        w.uniform_(-bb, bb)
    return w, torch.empty(fan_out, dtype=D).uniform_(-bb, bb)


def film():
    return 30 + 15 * 0.3 * torch.randn(H, dtype=D), 0.3 * torch.randn(H, dtype=D)


def q16(t):
    return t.to(torch.float16).to(D)


def split(t):
    hi = q16(t)
    return hi, q16(t - hi)


def mm(a, w, mode):
    if mode == "f64":
        return a @ w.t()
    if mode == "f16":
        return q16(a) @ q16(w).t()
    ah, al = split(a)
    wh, wl = split(w)
    return ah @ wh.t() + al @ wh.t() + ah @ wl.t()


def run(kind, m_trunk, m_bridge, m_c0, m_rest, scaled=False):
    torch.manual_seed(1)
    trunk = [lin(3, H, "first")] + [lin(H, H, "freq") for _ in range(7)]
    sig = lin(H, 1, "freq")
    if kind == "aug":
        bridge = lin(H, 3, "default")                   # color_layer_pre
        c0 = lin(6, H, "freq")
        ncol = 8
    else:
        bridge = lin(H, 3, "default")                   # res_coord_layer
        chain = [lin(3, H, "freq"), lin(H, H, "freq"), lin(H, H, "freq"), lin(H, 1, "freq")]
        cpre = lin(3, H, "default")
        c0 = lin(H + 3, H, "freq")
        ncol = 6
    crest = [lin(H, H, "freq") for _ in range(ncol - 1)]
    rgb = lin(H, 3, "freq")
    fl = [film() for _ in range(8 + ncol)]
    torch.manual_seed(2)
    pos = torch.rand(N, 3, dtype=D) * 2 - 1
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, dtype=D), dim=1)

    def layer(a, wb, fp, mode):
        return torch.sin(fp[0] * (mm(a, wb[0], mode) + wb[1]) + fp[1])

    x = pos
    for i, wb in enumerate(trunk):
        x = layer(x, wb, fl[i], "split" if i == 0 else m_trunk)
    v = mm(x, bridge[0], m_bridge) + bridge[1]
    if kind == "aug":
        sigma = mm(x, sig[0], m_trunk) + sig[1]
        c = layer(torch.cat([dirs, v], 1), c0, fl[8], m_c0)
    else:
        v = pos + v
        # the 4-Linear density chain and colour_layer_pre folded in float64 (affine maps)
        a, cst = chain[0]
        for w, b in chain[1:]:
            a, cst = w @ a, w @ cst + b
        if scaled:
            a, cst = a / a.abs().max(), cst * 0
        sigma = v @ a.t() + cst
        wf = c0[0][:, 3:] @ cpre[0]
        bf = c0[0][:, 3:] @ cpre[1] + c0[1]
        c = layer(torch.cat([dirs, v], 1), (torch.cat([c0[0][:, :3], wf], 1), bf), fl[8], m_c0)
    for j, wb in enumerate(crest):
        c = layer(c, wb, fl[9 + j], m_rest)
    out = torch.sigmoid(mm(c, rgb[0], m_rest) + rgb[1])
    return out, sigma, v


for kind, scaled in (("aug", False), ("res", False), ("res", True)):
    ref, sref, vref = run(kind, "f64", "f64", "f64", "f64", scaled)
    print(kind + (" (density chain scaled)" if scaled else ""), " |v| rms %.3f  |sigma| rms %.2e" % (vref.pow(2).mean().sqrt(), sref.pow(2).mean().sqrt()))
    for label, mt, mb, m0, mr in (("all fp16 (narrow colour 0 split)", "f16", "f16", "split", "f16"),
                                  ("bridge head split", "f16", "split", "split", "f16"),
                                  ("narrow colour 0 single fp16", "f16", "f16", "f16", "f16")):
        out, s, v = run(kind, mt, mb, m0, mr, scaled)
        d = (out - ref).abs()
        print("  %-34s v err max %.2e | sigma err max %.2e | rgb err max %.2e 99.9%% %.2e" % (
            label, (v - vref).abs().max(), (s - sref).abs().max(), d.max(), d.flatten().quantile(0.999)))
