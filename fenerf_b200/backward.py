"""Backward of the render: a ``torch.autograd.Function`` over the CUDA library (SURVEY.md section 8f-1).

What the reference differentiates (train_double_latent_semantic.py:405-446, the G step under autocast;
inverse_render_double_semantic.py:385-407, Adam on FiLM offsets through ``forward_with_frequencies``,
generators/generators.py:735-798): the final ``fancy_integration`` over the merged samples and both
point-network passes.  Ray set-up and resampling are ``no_grad`` there too (generators.py:41, 59).

forward   ONE ``fenerf_render_forward`` call into a private workspace -- the same kernels, numerics and
          precision modes as the no_grad path; the workspace (sample points, depths, raw field outputs of
          both passes) is what the backward needs and is kept alive by the autograd node.
backward  ``fenerf_composite_backward`` (d pixels -> d raw outputs, one warp per ray), then the point
          network layer by layer, recomputing activations chunk by chunk (nothing but the workspace
          survives from the forward):
            recompute   ``fenerf_gemm_nt_film``: z = a W^T on wgmma with the epilogue fused -- a = sin(f z + p) and
                        the gate cos(f z + p) leave as fp16, z never does
            backward    ``fenerf_gate_backward`` dU = dA * gate = dL/du (+ per-image column sums dp_b),
                        dA' = dU diag(f_b) W (``fenerf_gemm_nt_f16`` with a per-image scaled weight, one launch per
                        image of the chunk) and the per-image M_b = dU_b^T a (``fenerf_gemm_tn_f16``, split-K)
          Every gradient of the layer follows from M_b and dp_b without another pass over the points, and none divides
          by f (a frequency of exactly 0 is reachable from the mapping network's 15 x + 30):
          dW = sum_b diag(f_b) M_b,  db = sum_b f_b dp_b,  df_b = rowsum(W * M_b) + b dp_b   (u = f z + p, z = W a + b).
          Heads, the pre-multiplied label chain and the grid (``fenerf_grid_scatter_add``, from the first colour layer's
          dU, or from the first layer's where the grid feeds the trunk, EmbeddingPiGAN256) close the chain.  A label FiLM
          field (SPATIALSIRENSEMANTIC) recomputes its label layer from the trunk output at FiLM row T and runs it
          backward like a colour layer, its dU diag(f) W joining the trunk's dA.  A bridge field (SPATIALSIRENAUGDISENTANGLE,
          RESSIRENDISENTANGLE) recomputes v = W_v a + b_v (+ the position) off the trunk output and its first colour layer
          from [dir, v] like a first layer; dv = dU diag(f) W_c0[:, v] (+ dsigma a for RES) joins the trunk as dv W_v:
          dU diag(f_b) (W_c0[:, v] W_v) through the same per-image product as every other layer, and for RES dsigma a W_v
          as the trunk's sigma head.  A skinny library product for dv would give each row fp32 values that depend on the
          chunk's row count, and the fp16 dA would round them differently from chunk layout to chunk layout.  The
          direction-free field (TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96) runs as a grid field whose
          first colour layer has zero direction columns (finish() drops them from its weight gradient), in the exact
          mode only: that layer's U(+-1/3) weights at f ~ 30 amplify the fp16 streams' error past any useful bound.
Gradients flow to the FiLM table (and through torch's autograd into the mapping network / latents /
frequency offsets) and to every field parameter.  The fp16 gradient stream is scaled by a power of two
taken from max|d raw| on the device (no host sync) and unscaled at the end.

The three 256-wide products per layer run on wgmma (csrc/gemm.cu: ``fenerf_gemm_nt_film`` -- the recompute with its FiLM
epilogue fused, ``fenerf_gemm_nt_f16`` for dA' = dU diag(f_b) W, ``fenerf_gemm_tn_f16`` split-K for the per-image M_b); only the narrow
products (heads, the 3 / 35-wide inputs) go to the library.  ``FENERF_B200_BWD_GEMM=cublas`` switches the wide ones back
(A/B timing); ``precision='exact'`` uses fp32 library GEMMs, or, with ``grad_precision='split'``, the split kernels of
csrc/gemm_split.cu on the same fp32 streams (fp16 hi / lo operands scaled by powers of two, fp32-grade results).  (The kernels can also fold the next layer's gate multiply
into the dA product's epilogue and produce the bias column sums from the dW kernel's staged tiles -- measured: the gate kernel's
17 ms disappear but the two GEMMs slow down by as much, both being HBM-bound; the chain below keeps the separate gate kernel.)
"""
import ctypes as C

import torch

from . import _lib, ops, packing

import os

CHUNK_POINTS = 1 << 19
#: the 256-wide products: 'wgmma' = csrc/gemm.cu (default), 'cublas' = torch.mm / bmm (kept for A/B timing and as the
#: fp32 path of precision='exact')
BWD_GEMM = os.environ.get("FENERF_B200_BWD_GEMM", "wgmma")


def _ptr(t):
    return t.data_ptr() if t is not None else 0


def _stream(device):
    return torch.cuda.current_stream(device).cuda_stream


def _mm32(a, b):
    """fp16 x fp16 -> fp32 (tensor cores, fp32 accumulate AND fp32 output); plain fp32 in the exact mode."""
    if a.dtype == torch.float32:
        return torch.mm(a, b)
    return torch.mm(a, b, out_dtype=torch.float32)


class _NoTF32:
    """Keeps torch's fp32 products fp32 (no TF32) inside the block, whatever the caller's matmul switch says."""

    def __enter__(self):
        self.prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cuda.matmul.allow_tf32 = self.prev


def _bmm32(a, b):
    if a.dtype == torch.float32:
        return torch.bmm(a, b)
    return torch.bmm(a, b, out_dtype=torch.float32)


class FieldWeights:
    """The field's parameters in the roles the backward needs, plus fp16 copies for the GEMMs."""

    def __init__(self, module):
        spec = module.field_spec()
        self.spec = spec
        net = list(module.network)
        color = module.color_layer_sine
        color = list(color) if isinstance(color, torch.nn.ModuleList) else [color]
        self.trunk = [(l.layer.weight, l.layer.bias) for l in net]
        self.color = [(l.layer.weight, l.layer.bias) for l in color]
        # (RESSIRENDISENTANGLE has no final_layer: its density is the chain on v)
        self.sigma = None if spec.bridge_res else (module.final_layer.weight, module.final_layer.bias)
        # a bridge field's v = Linear(256 -> 3) of the trunk output, its density chain and color_layer_pre (RES)
        self.bridge = None
        if spec.bridge:
            lin = module.res_coord_layer if spec.bridge_res else module.color_layer_pre[0]
            self.bridge = (lin.weight, lin.bias)
        self.density = [(m.weight, m.bias) for m in module.density_layer_linear] if spec.bridge_res else []
        self.pre = (module.color_layer_pre[0].weight, module.color_layer_pre[0].bias) if spec.bridge_res else None
        self.rgb = (module.color_layer_linear[0].weight, module.color_layer_linear[0].bias)
        self.labels = []
        if spec.label_dim:
            self.labels = [(m.weight, m.bias) for m in module.label_layer_linear if isinstance(m, torch.nn.Linear)]
        # the label FiLM layer (FiLM row len(trunk)); self.labels is then its one-Linear head
        self.label_film = [(module.label_layer_sine.layer.weight, module.label_layer_sine.layer.bias)] if spec.label_film else []
        self.grid = module.spatial_embeddings if spec.grid_channels else None

    def film_layers(self):
        """(weight, bias) of every FiLM layer in FiLM-table row order: trunk, label FiLM layer, colour."""
        return self.trunk + self.label_film + self.color

    def parameters(self):
        ps = []
        extra = [self.sigma] if self.sigma is not None else []
        extra += ([self.bridge] if self.bridge is not None else []) + self.density + ([self.pre] if self.pre else [])
        for w, b in self.film_layers() + extra + [self.rgb] + self.labels:
            ps += [w, b]
        if self.grid is not None:
            ps.append(self.grid)
        return ps


def _label_eff(labels):
    """Weff, beff of the activation-free label chain (siren.py:1486-1490 / 1189-1191), fp32 via fp64."""
    ws = [w.detach().double() for w, _ in labels]
    bs = [b.detach().double() for _, b in labels]
    if len(labels) == 3:
        u = ws[2] @ ws[1]
        return (u @ ws[0]).float(), (u @ bs[0] + ws[2] @ bs[1] + bs[2]).float()
    return (ws[1] @ ws[0]).float(), (ws[1] @ bs[0] + bs[1]).float()


def _label_chain_grads(labels, d_weff, d_beff):
    """Gradients of the chain's own parameters from those of the pre-multiplied map."""
    ws = [w.detach().double() for w, _ in labels]
    bs = [b.detach().double() for _, b in labels]
    dw, db = d_weff.double(), d_beff.double()
    if len(labels) == 3:
        w1, w2, w3 = ws
        b1, b2, _ = bs
        u = w3 @ w2
        g1w, g1b = u.t() @ dw, u.t() @ db
        g2w = w3.t() @ (dw @ w1.t() + torch.outer(db, b1))
        g2b = w3.t() @ db
        g3w = dw @ (w2 @ w1).t() + torch.outer(db, w2 @ b1 + b2)
        return [(g1w, g1b), (g2w, g2b), (g3w, db)]
    w1, w3 = ws
    b1, _ = bs
    return [(w3.t() @ dw, w3.t() @ db), (dw @ w1.t() + torch.outer(db, b1), db)]


def _linear_chain_eff(chain):
    """Weff, beff of an activation-free chain of Linears (first applied first), in fp64."""
    weff, beff = None, None
    for w, b in chain:
        w, b = w.detach().double(), b.detach().double()
        weff, beff = (w, b) if weff is None else (w @ weff, w @ beff + b)
    return weff, beff


def _linear_chain_grads(chain, d_weff, d_beff):
    """Gradients of every Linear of an activation-free chain from those of its product map (fp64; RESSIRENDISENTANGLE's
    density_layer_linear): layer i sees dW_i = U_i^T (dWeff R_i^T + dbeff s_i^T), db_i = U_i^T dbeff, with U_i the
    product of the layers after it, R_i the one before it and s_i the bias that reaches its input."""
    ws = [w.detach().double() for w, _ in chain]
    bs = [b.detach().double() for _, b in chain]
    dw, db = d_weff.double(), d_beff.double()
    out = []
    for i in range(len(chain)):
        u = torch.eye(ws[i].shape[0], dtype=torch.float64, device=dw.device)
        for w in ws[i + 1:]:
            u = w @ u
        r = torch.eye(ws[0].shape[1], dtype=torch.float64, device=dw.device)
        s_in = torch.zeros(ws[0].shape[1], dtype=torch.float64, device=dw.device)
        for w, b in zip(ws[:i], bs[:i]):
            r, s_in = w @ r, w @ s_in + b
        out.append((u.t() @ (dw @ r.t() + torch.outer(db, s_in)), u.t() @ db))
    return out


#: the render keyword ``grad_precision``: None (the backward of the forward precision) or 'split'
GRAD_PRECISIONS = (None, "split")
_GRAD_SPLIT_STREAMS = ("grad_precision='split' differentiates precision='split' or 'exact' renders only: it runs on their "
                       "fp32 streams (precision='fast' / 'guard' keep the fp16 backward)")


def _grad_split_refusal(spec):
    """Why grad_precision='split' cannot differentiate a field of this spec (None: it can).  The same variants as the split
    forward (FENERF_PRECISION_SPLIT) refuses."""
    kinds = [name for name, on in (("a label FiLM layer", spec.label_film), ("a feature head", spec.feature_head),
                                   ("grid features in the trunk", spec.grid_trunk), ("a bridge colour branch", spec.bridge))
             if on]
    if not kinds:
        return None
    return ("grad_precision='split' is not built for fields with %s (FENERF_FIELD_LABEL_FILM, FENERF_FIELD_FEATURE_HEAD, "
            "FENERF_FIELD_GRID_TRUNK, FENERF_FIELD_BRIDGE); differentiate them without grad_precision" % " and ".join(kinds))


def check_grad_precision(module, grad_precision, precision):
    """Raises unless a differentiable render of `module` in forward precision `precision` (name or code) can take
    `grad_precision`: ValueError for an unknown name, RuntimeError with the reason for a refused combination."""
    if grad_precision not in GRAD_PRECISIONS:
        raise ValueError("grad_precision must be one of %s (got %r)" % (GRAD_PRECISIONS, grad_precision))
    if grad_precision is None:
        return
    if ops._precision_code(precision) not in (_lib.PRECISION["split"], _lib.PRECISION["exact"]):
        raise RuntimeError(_GRAD_SPLIT_STREAMS)
    reason = _grad_split_refusal(module.field_spec())
    if reason:
        raise RuntimeError(reason)


class _FieldBackward:
    """Accumulates the gradients of one field over any number of point sets."""

    def __init__(self, module, film, scale, inv_scale, exact=False, split=False, grad_split=False):
        self.module = module
        # grad_split (grad_precision='split'): the fp32 streams of the exact mode, the 256-wide products on the split
        # kernels of csrc/gemm_split.cu
        self.gs = bool(grad_split)
        if self.gs and not exact:
            raise RuntimeError(_GRAD_SPLIT_STREAMS)
        if self.gs and _grad_split_refusal(module.field_spec()):
            raise RuntimeError(_grad_split_refusal(module.field_spec()))
        # stream element type: fp16 (default) or fp32 (parity mode, with precision='exact': plain fp32 GEMMs)
        self.dt = torch.float32 if exact else torch.float16
        self.dtc = 1 if exact else 0
        self.fw = FieldWeights(module)
        self.spec = self.fw.spec
        self.packed = module.packed(split=split)       # (split: the pack the forward rendered from; same sections)
        self.film = film.detach().float().contiguous()           # (B, n_film, 2, 256)
        self.scale, self.inv_scale = scale, inv_scale
        dev = self.film.device
        self.dev = dev
        B = self.film.shape[0]
        T, Cn = len(self.fw.trunk), len(self.fw.color)
        self.lf = len(self.fw.label_film)                          # 1: a label FiLM layer at row T, colour from T + 1
        self.T, self.Cn, self.c0, self.n_film = T, Cn, T + self.lf, T + self.lf + Cn
        G = self.spec.grid_channels
        # narrow inputs: the first layer's [pos] -- [feat, pos] with the grid in the trunk (EmbeddingPiGAN256) -- and the
        # first colour layer's [dir, feat] -- [dir] with the grid in the trunk
        self.gt = self.spec.grid_trunk
        self.k0 = 3 + G if self.gt else 3
        self.k0_pad = (self.k0 + 7) // 8 * 8
        self.br, self.res = self.spec.bridge, self.spec.bridge_res
        self.kx = 3 if self.gt else 6 if self.br else 3 + G
        self.kx_pad = (self.kx + 7) // 8 * 8
        # per-image accumulators (scaled by `scale`)
        self.colsum = torch.zeros((B, self.n_film, 256), dtype=torch.float32, device=dev)
        self.dW_b = [None] * self.n_film
        self.dW_b[0] = torch.zeros((B, 256, self.k0_pad), dtype=torch.float32, device=dev)
        for i in range(1, self.n_film):
            self.dW_b[i] = torch.zeros((B, 256, 256), dtype=torch.float32, device=dev)
        self.dWx_b = torch.zeros((B, 256, self.kx_pad), dtype=torch.float32, device=dev)   # colour 0's narrow inputs
        # head-gradient widths of fenerf_head_grads: [labels, sigma, pad] and the colour head's (include/fenerf_b200.h)
        L = self.spec.label_dim
        self.n_heads = L + 8 if self.spec.feature_head else 32
        self.n_rgb = 64 if self.spec.feature_head else 8
        self.d_heads_w = torch.zeros((self.n_heads, 256), dtype=torch.float32, device=dev)
        self.d_heads_b = torch.zeros((self.n_heads,), dtype=torch.float32, device=dev)
        self.d_rgb_w = torch.zeros((self.n_rgb, 256), dtype=torch.float32, device=dev)
        self.d_rgb_b = torch.zeros((self.n_rgb,), dtype=torch.float32, device=dev)
        self.grid_grad_cl = None
        if G:
            r = self.spec.grid_res
            self.grid_grad_cl = torch.zeros((r, r, r, G), dtype=torch.float32, device=dev)
        # torch.use_deterministic_algorithms(True): the column sums and the grid scatter in a fixed order
        # (csrc/backward_det.cu) instead of float atomics; the fixed-point grid scatter's workspace (2.5x the accumulator)
        self.det = torch.are_deterministic_algorithms_enabled()
        self.grid_det_ws = None
        if G and self.det:
            nbytes = _lib.lib().fenerf_grid_scatter_det_workspace_bytes(C.byref(self.packed.desc))
            self.grid_det_ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        # fp16 / fp32 weight views for the GEMMs
        fw = self.fw
        self.W0 = fw.trunk[0][0].detach().float().contiguous()                    # (256, 3); grid trunk (256, G + 3)
        self.own_gemm = (not exact) and BWD_GEMM == "wgmma"
        self.Wh16 = [None] + [w.detach().to(self.dt).contiguous() for w, _ in fw.trunk[1:]]
        wc0 = fw.color[0][0].detach().float()
        # a direction-free field's first colour layer reads [feat, x]: zero direction columns give it the [dir, feat, x]
        # order of the other grid fields (finish() drops them again)
        self.wd = self.spec.wo_dir
        if self.wd and not exact:
            raise RuntimeError("the direction-free field (FENERF_FIELD_WO_DIR) renders and differentiates in "
                               "precision='exact' only: its first colour layer amplifies the fp16 streams' error (precision='split' "
                               "renders it on the tensor cores and differentiates as 'exact')")
        if self.wd:
            wc0 = torch.cat([torch.zeros((256, 3), dtype=torch.float32, device=dev), wc0], dim=1)
        self.bias = [b.detach().float().contiguous() for _, b in fw.film_layers()]
        if self.br:
            # the first colour layer on [dir, v]; RES: color_layer_pre folded into its v columns and bias (fp64)
            wc0d = fw.color[0][0].detach().double()
            if self.res:
                pw, pb = (t.detach().double() for t in fw.pre)
                self.Wc0eff = torch.cat([wc0d[:, :3], wc0d[:, 3:] @ pw], dim=1).float().contiguous()
                self.bias[self.c0] = (fw.color[0][1].detach().double() + wc0d[:, 3:] @ pb).float().contiguous()
                a, c = _linear_chain_eff(fw.density)
                self.dens_a, self.dens_c = a.float().reshape(3), c.float().reshape(())
                self.d_a = torch.zeros(3, dtype=torch.float32, device=dev)
                self.d_c = torch.zeros((), dtype=torch.float32, device=dev)
            else:
                self.Wc0eff = wc0.contiguous()
            self.Wv32 = fw.bridge[0].detach().float().contiguous()                  # (3, 256)
            self.bv32 = fw.bridge[1].detach().float().contiguous()
            self.d_wv = torch.zeros((3, 256), dtype=torch.float32, device=dev)
            self.d_bv = torch.zeros(3, dtype=torch.float32, device=dev)
            wc0 = torch.cat([self.Wc0eff, torch.zeros((256, 256), dtype=torch.float32, device=dev)], dim=1)
        self.Wc0x_narrow = wc0[:, :self.kx].contiguous()                          # (256, 3 + G) fp32
        self.Wc16 = [wc0[:, self.kx:].to(self.dt).contiguous()] + [w.detach().to(self.dt).contiguous() for w, _ in fw.color[1:]]
        # grad_split: the recompute's 256-wide weights by FiLM row (trunk 1.., colour c0..), split as (hi, lo, amax)
        self.Wsplit = [None] + [ops.split_weights(w) for w in self.Wh16[1:] + self.Wc16] if self.gs else None
        # the weights the grid features meet, (256, G): the first colour layer's, or the first layer's with the grid in
        # the trunk, whose FiLM row is then 0
        self.feat_row = 0 if self.gt else self.c0
        self.Wfeat32 = (self.W0[:, :G] if self.gt else wc0[:, 3:self.kx].contiguous()) if G else None
        # fp32 weights of the chain products dA' = dU diag(f_b) W, by FiLM row (row 0 has none: its inputs are the points)
        self.Wchain32 = [None] + [w.detach().float() for w, _ in fw.trunk[1:]]
        if self.lf:
            self.Wl16 = fw.label_film[0][0].detach().to(self.dt).contiguous()
            self.Wchain32.append(fw.label_film[0][0].detach().float())
            self.Wlhead32 = fw.labels[0][0].detach().float().contiguous()                 # (L, 256)
        # a bridge field's first colour layer passes dU diag(f_b) W_c0[:, v] W_v (rank 3) to the trunk
        wc0_chain = (self.Wc0eff[:, 3:6].double() @ self.Wv32.double()).float() if self.br else wc0[:, self.kx:]
        self.Wchain32 += [wc0_chain] + [w.detach().float() for w, _ in fw.color[1:]]
        # ... scaled per image once for every chunk: diag(f_b) W, (B, n_film - 1, 256, 256); the NT kernel wants it transposed
        fW = self.film[:, 1:, 0].unsqueeze(3) * torch.stack(self.Wchain32[1:])
        if self.gs:     # per image and layer, (diag(f_b) W)^T scaled by its own power of two and split
            self.fW_hi, self.fW_lo, self.fW_amax = ops.split_weights(fW.transpose(2, 3))
            self.fW = None
        else:
            self.fW = fW.transpose(2, 3).to(torch.float16).contiguous() if self.own_gemm else fW.to(self.dt)
        del fW
        self.fWfeat = (self.film[:, self.feat_row, 0].unsqueeze(2) * self.Wfeat32).to(self.dt) if G else None    # (B, 256, G)
        if self.own_gemm:
            self.Wn64 = torch.zeros((256, 64), dtype=torch.float16, device=dev)
            self.Wn64[:, :self.kx] = self.Wc0x_narrow
        self.L = L
        heads = torch.zeros((self.n_heads, 256), dtype=torch.float32, device=dev)
        if L and not self.lf:      # (a label FiLM field's head acts on the label layer: its rows stay zero here)
            weff, _ = _label_eff(fw.labels)
            heads[:L] = weff
        if fw.sigma is not None:
            heads[L] = fw.sigma[0].detach().float().reshape(-1)
        elif self.res:                 # sigma = a . v + c with v = W_v h + ...: the trunk's sigma head is a W_v
            heads[L] = (self.dens_a.double() @ self.Wv32.double()).float()
        self.Wheads32 = heads
        rgbw = torch.zeros((self.n_rgb, 256), dtype=self.dt, device=dev)
        rgbw[:self.spec.rgb_dim] = fw.rgb[0].detach().to(self.dt)
        self.Wrgb16 = rgbw

    # ---- one point set: points (B, ppb, 3), dirs (B, ppb/dir_group, 3), raw / d_raw (B, ppb, C) ----
    def add_points(self, points, dirs, dir_group, lock_dirs, raw, d_raw):
        if self.wd or self.gs:     # the direction-free field: TF32 rounding would be amplified like fp16's (see __init__);
            with _NoTF32():          # grad_split: its narrow products stay fp32
                return self._add_points(points, dirs, dir_group, lock_dirs, raw, d_raw)
        return self._add_points(points, dirs, dir_group, lock_dirs, raw, d_raw)

    def _add_points(self, points, dirs, dir_group, lock_dirs, raw, d_raw):
        B, ppb, _ = points.shape
        if ppb <= CHUNK_POINTS:
            k = max(1, CHUNK_POINTS // ppb)
            for b0 in range(0, B, k):
                b1 = min(B, b0 + k)
                self._chunk(points[b0:b1], dirs[b0:b1], dir_group, lock_dirs, raw[b0:b1], d_raw[b0:b1], b0, b1)
        else:
            step = CHUNK_POINTS // dir_group * dir_group
            for b in range(B):
                for p0 in range(0, ppb, step):
                    p1 = min(ppb, p0 + step)
                    self._chunk(points[b:b + 1, p0:p1], dirs[b:b + 1, p0 // dir_group:p1 // dir_group], dir_group, lock_dirs,
                                raw[b:b + 1, p0:p1], d_raw[b:b + 1, p0:p1], b, b + 1)

    def _stash(self, z, idx, b0, P, ppb, xin=None, wx=None):
        a = torch.empty((P, 256), dtype=self.dt, device=self.dev)
        g = torch.empty((P, 256), dtype=self.dt, device=self.dev)
        film_l = self.film[b0, idx]
        kx = 0 if xin is None else xin.shape[1]
        _lib.check(_lib.lib().fenerf_film_forward_stash(
            _ptr(z), self.bias[idx].data_ptr(), film_l.data_ptr(), self.film.stride(0), P, ppb,
            _ptr(xin), kx, _ptr(wx), a.data_ptr(), g.data_ptr(), self.dtc, _stream(self.dev)))
        return a, g

    def _gate(self, dA, gate, idx, b0, b1, P, ppb):
        cs = self.colsum[b0:b1, idx]
        tmp = torch.zeros((b1 - b0, 256), dtype=torch.float32, device=self.dev)
        if self.det:     # each 512-point slab's sums to its own row, added in a fixed order
            part = torch.empty(P // ppb * ((ppb + 511) // 512) * 256, dtype=torch.float32, device=self.dev)
            _lib.check(_lib.lib().fenerf_gate_backward_det(dA.data_ptr(), gate.data_ptr(), P, ppb, part.data_ptr(),
                                                           part.numel() * 4, tmp.data_ptr(), self.dtc, _stream(self.dev)))
        else:
            _lib.check(_lib.lib().fenerf_gate_backward(dA.data_ptr(), gate.data_ptr(), P, ppb, tmp.data_ptr(), self.dtc,
                                                       _stream(self.dev)))
        cs += tmp

    def _chain(self, dU, idx, b0, b1, ppb, amax=None):
        """dU diag(f_b) W of FiLM row idx for each image b of the chunk: the gradient of the layer's input (P, 256).
        amax: max |dU| on the device (grad_split)."""
        k = b1 - b0
        if self.gs:
            out = torch.empty_like(dU)
            for i in range(k):
                rows = slice(i * ppb, (i + 1) * ppb)
                ops.gemm_nt_split(dU[rows], self.fW_hi[b0 + i, idx - 1], self.fW_lo[b0 + i, idx - 1],
                                  self.fW_amax[b0 + i, idx - 1], a_amax=amax, out=out[rows])
            return out
        if not self.own_gemm:
            return torch.bmm(dU.view(k, ppb, 256), self.fW[b0:b1, idx - 1]).view(k * ppb, 256)
        out = torch.empty_like(dU)
        for i in range(k):
            rows = slice(i * ppb, (i + 1) * ppb)
            ops.gemm_nt(dU[rows], self.fW[b0 + i, idx - 1], torch.float16, out=out[rows])
        return out

    def _chunk(self, points, dirs, dir_group, lock_dirs, raw, d_raw, b0, b1):
        lib = _lib.lib()
        dev, spec = self.dev, self.spec
        k, ppb = points.shape[0], points.shape[1]
        P = k * ppb
        T, Cn, c0 = self.T, self.Cn, self.c0
        points = points.contiguous()
        dirs = dirs.contiguous()
        raw = raw.contiguous()
        d_raw = d_raw.contiguous()
        with torch.cuda.device(dev):
            st = _stream(dev)
            # ---- recompute the forward, stashing activations and gates (fp16) ----
            x = (points.reshape(P, 3) * spec.input_scale).contiguous() if spec.input_scale != 1.0 else points.reshape(P, 3)
            G = spec.grid_channels
            extras = torch.empty((P, 3 + G), dtype=torch.float32, device=dev)     # [dir, feat]
            _lib.check(lib.fenerf_extras_gather(C.byref(self.packed.desc), self.packed.ptr, points.data_ptr(), dirs.data_ptr(),
                                                P, ppb, dir_group, int(bool(lock_dirs)), extras.data_ptr(), st))
            if self.gt:     # the first layer takes [feat, pos] (the reference's column order), the colour layer [dir]
                x = torch.cat([extras[:, 3:], x], dim=1).contiguous()
                extras = extras[:, :3].contiguous()
            A, Gt = [None] * self.n_film, [None] * self.n_film
            own = self.own_gemm
            A[0], Gt[0] = self._stash(None, 0, b0, P, ppb, xin=x, wx=self.W0)
            for l in range(1, T):
                if own:     # z = a W^T with the FiLM epilogue fused: z never leaves the SM
                    A[l], Gt[l] = ops.gemm_nt_film(A[l - 1], self.Wh16[l], self.bias[l], self.film, b0, l, ppb)
                elif self.gs:
                    A[l], Gt[l] = ops.gemm_nt_film_split(A[l - 1], *self.Wsplit[l], self.bias[l], self.film, b0, l, ppb)
                else:
                    A[l], Gt[l] = self._stash(_mm32(A[l - 1], self.Wh16[l].t()), l, b0, P, ppb)
            if self.lf:     # the label FiLM layer, on the trunk output
                if own:
                    A[T], Gt[T] = ops.gemm_nt_film(A[T - 1], self.Wl16, self.bias[T], self.film, b0, T, ppb)
                else:
                    A[T], Gt[T] = self._stash(_mm32(A[T - 1], self.Wl16.t()), T, b0, P, ppb)
            v = None
            if self.br:     # v off the trunk output (fp32), then the first colour layer on [dir, v] like a first layer
                v = _mm32(A[T - 1], self.Wv32.t().to(self.dt)) + self.bv32
                if self.res:
                    v = v + x
                extras = torch.cat([extras, v], dim=1).contiguous()
                A[c0], Gt[c0] = self._stash(None, c0, b0, P, ppb, xin=extras, wx=self.Wc0eff)
            elif own:     # the narrow inputs [dir, grid features] ride as a fifth 64-wide k-chunk of the same kernel
                e64 = torch.zeros((P, 64), dtype=torch.float16, device=dev)
                e64[:, :self.kx] = extras
                A[c0], Gt[c0] = ops.gemm_nt_film(A[T - 1], self.Wc16[0], self.bias[c0], self.film, b0, c0, ppb, narrow_in=e64,
                                                 narrow_w=self.Wn64)
                del e64
            else:
                z = ops.gemm_nt_split(A[T - 1], *self.Wsplit[c0]) if self.gs else _mm32(A[T - 1], self.Wc16[0].t())
                A[c0], Gt[c0] = self._stash(z, c0, b0, P, ppb, xin=extras, wx=self.Wc0x_narrow)
                del z
            for j in range(1, Cn):
                if own:
                    A[c0 + j], Gt[c0 + j] = ops.gemm_nt_film(A[c0 + j - 1], self.Wc16[j], self.bias[c0 + j], self.film, b0, c0 + j,
                                                             ppb)
                elif self.gs:
                    A[c0 + j], Gt[c0 + j] = ops.gemm_nt_film_split(A[c0 + j - 1], *self.Wsplit[c0 + j], self.bias[c0 + j], self.film,
                                                                   b0, c0 + j, ppb)
                else:
                    A[c0 + j], Gt[c0 + j] = self._stash(_mm32(A[c0 + j - 1], self.Wc16[j].t()), c0 + j, b0, P, ppb)
            # ---- head gradients ----
            dH = torch.empty((P, self.n_heads), dtype=self.dt, device=dev)
            dRGB = torch.empty((P, self.n_rgb), dtype=self.dt, device=dev)
            _lib.check(lib.fenerf_head_grads(d_raw.data_ptr(), raw.data_ptr(), P, spec.out_dim, self.L, self.scale.data_ptr(),
                                             dH.data_ptr(), dRGB.data_ptr(), self.dtc, st))
            a_last = A[self.n_film - 1]
            d_sigma = dH[:, self.L].float()
            self.d_rgb_w += _mm32(dRGB.t(), a_last)
            self.d_rgb_b += dRGB.float().sum(0)
            if self.lf:     # label rows on the label layer's activations, the sigma row on the trunk's
                L = self.L
                self.d_heads_w[:L] += _mm32(dH[:, :L].t(), A[T])
                self.d_heads_w[L:] += _mm32(dH[:, L:].t(), A[T - 1])
            else:
                self.d_heads_w += _mm32(dH.t(), A[T - 1])
            self.d_heads_b += dH.float().sum(0)
            # ---- colour branch, top down ----
            dA = torch.mm(dRGB, self.Wrgb16)                                   # (P, 256) fp16
            for j in range(Cn - 1, -1, -1):
                idx = c0 + j
                self._gate(dA, Gt[idx], idx, b0, b1, P, ppb)                   # dA is dU now
                if self.br and j == 0:
                    self._bridge_back(dA, extras, v, A[T - 1], d_sigma, k, ppb, b0, b1)
                    dA = self._chain(dA, idx, b0, b1, ppb)
                    A[idx], Gt[idx] = None, None
                    break
                a_in = A[idx - 1] if j else A[T - 1]
                du3 = dA.view(k, ppb, 256).transpose(1, 2)
                amax = ops.absmax(dA) if self.gs else None      # (grad_split: the scale of this layer's dU, on the device)
                if self.gs:
                    self.dW_b[idx][b0:b1] += ops.gemm_tn_split(dA, a_in, k, ppb, x_amax=amax)
                else:
                    self.dW_b[idx][b0:b1] += ops.gemm_tn(dA, a_in, k, ppb) if own else _bmm32(du3, a_in.view(k, ppb, 256))
                if j == 0:
                    e16 = torch.zeros((P, self.kx_pad), dtype=self.dt, device=dev)
                    e16[:, :self.kx] = extras
                    self.dWx_b[b0:b1] += _bmm32(du3, e16.view(k, ppb, self.kx_pad))
                    if G and not self.gt:
                        self._grid_grad(dA, points, k, ppb, b0, b1)
                dA = self._chain(dA, idx, b0, b1, ppb, amax)
                A[idx], Gt[idx] = None, None
            # ---- trunk: colour-branch gradient + sigma / label heads ----
            dA += torch.mm(dH.float(), self.Wheads32)
            if self.lf:     # label branch: d logits W_head -> gate -> M_b, colsum of row T; dU diag(f) W_label joins the trunk's dA
                # (P, 256), formed in fp32: an fp16 product's reduction order depends on the chunk's row count
                dAl = torch.mm(dH[:, :self.L].float(), self.Wlhead32).to(self.dt)
                self._gate(dAl, Gt[T], T, b0, b1, P, ppb)
                if own:
                    self.dW_b[T][b0:b1] += ops.gemm_tn(dAl, A[T - 1], k, ppb)
                else:
                    self.dW_b[T][b0:b1] += _bmm32(dAl.view(k, ppb, 256).transpose(1, 2), A[T - 1].view(k, ppb, 256))
                dA += self._chain(dAl, T, b0, b1, ppb)
                A[T], Gt[T] = None, None
            for l in range(T - 1, 0, -1):
                self._gate(dA, Gt[l], l, b0, b1, P, ppb)
                amax = ops.absmax(dA) if self.gs else None
                if own:
                    self.dW_b[l][b0:b1] += ops.gemm_tn(dA, A[l - 1], k, ppb)
                elif self.gs:
                    self.dW_b[l][b0:b1] += ops.gemm_tn_split(dA, A[l - 1], k, ppb, x_amax=amax)
                else:
                    self.dW_b[l][b0:b1] += _bmm32(dA.view(k, ppb, 256).transpose(1, 2), A[l - 1].view(k, ppb, 256))
                dA = self._chain(dA, l, b0, b1, ppb, amax)
                A[l], Gt[l] = None, None
            self._gate(dA, Gt[0], 0, b0, b1, P, ppb)
            if self.gt:
                self._grid_grad(dA, points, k, ppb, b0, b1)
            x16 = torch.zeros((P, self.k0_pad), dtype=self.dt, device=dev)
            x16[:, :self.k0] = x
            self.dW_b[0][b0:b1] += _bmm32(dA.view(k, ppb, 256).transpose(1, 2), x16.view(k, ppb, self.k0_pad))

    def _bridge_back(self, dU, extras, v, a_trunk, d_sigma, k, ppb, b0, b1):
        """First colour layer of a bridge field on [dir, v]: its narrow weight gradient, dv = dU diag(f) W_c0[:, v]
        (+ dsigma a for RES) and v's own gradients, in fp32 (3 columns).  The trunk's share dv W_v goes through _chain
        and the sigma head instead (see the module docstring)."""
        P = k * ppb
        du = dU.float().view(k, ppb, 256)
        e = torch.zeros((P, self.kx_pad), dtype=torch.float32, device=self.dev)
        e[:, :self.kx] = extras
        self.dWx_b[b0:b1] += torch.bmm(du.transpose(1, 2), e.view(k, ppb, self.kx_pad))
        fwv = self.film[b0:b1, self.c0, 0].unsqueeze(2) * self.Wc0eff[:, 3:6]      # (k, 256, 3), no division by f
        dv = torch.bmm(du, fwv).view(P, 3)
        if self.res:
            dv = dv + d_sigma.unsqueeze(1) * self.dens_a
            self.d_a += (d_sigma.unsqueeze(1) * v).sum(0)
            self.d_c += d_sigma.sum()
        self.d_wv += dv.t() @ a_trunk.float()
        self.d_bv += dv.sum(0)

    def _grid_grad(self, dU, points, k, ppb, b0, b1):
        """d features = dU diag(f_b) W_feat, (P, G), of the layer the grid feeds, scattered into the grid accumulator."""
        P = k * ppb
        d_feat = torch.bmm(dU.view(k, ppb, 256), self.fWfeat[b0:b1]).view(P, -1).contiguous()
        if self.det:     # 64-bit fixed point at a scale taken from this point set's max |d feat|, integer atomics
            ws = self.grid_det_ws
            _lib.check(_lib.lib().fenerf_grid_scatter_add_det(C.byref(self.packed.desc), points.data_ptr(), d_feat.data_ptr(),
                                                              d_feat.shape[1], P, ws.data_ptr(), ws.numel(),
                                                              self.grid_grad_cl.data_ptr(), self.dtc, _stream(self.dev)))
            return
        _lib.check(_lib.lib().fenerf_grid_scatter_add(C.byref(self.packed.desc), points.data_ptr(), d_feat.data_ptr(),
                                                      d_feat.shape[1], P, self.grid_grad_cl.data_ptr(), self.dtc,
                                                      _stream(self.dev)))

    # ---- after every point set: fold the per-image accumulators into parameter / FiLM gradients ----
    def finish(self):
        if self.wd or self.gs:
            with _NoTF32():
                return self._finish()
        return self._finish()

    def _finish(self):
        fw, inv = self.fw, self.inv_scale
        film = self.film
        d_film = torch.zeros_like(film)
        grads = {}
        layers = fw.film_layers()
        for idx, (w, b) in enumerate(layers):
            f = film[:, idx, 0]                                             # (B, 256)
            dp = self.colsum[:, idx]                                        # sum of dU per image
            w32 = w.detach().float()
            if idx == 0:
                m = self.dW_b[0][:, :, :self.k0]                                # columns [pos], or [feat, pos]
            elif idx == self.c0 and self.br:
                m = self.dWx_b[:, :, :self.kx]                                  # [dir, v]
                w32 = self.Wc0eff                                               # (RES: color_layer_pre folded in)
            elif idx == self.c0:
                m = torch.cat([self.dWx_b[:, :, :self.kx], self.dW_b[idx]], dim=2)   # column order of the reference: [dir, feat, x]
                if self.wd:
                    w32 = torch.cat([torch.zeros_like(w32[:, :3]), w32], dim=1)    # [feat, x] with zero direction columns
            else:
                m = self.dW_b[idx]                                          # M_b = dU_b^T a
            df = torch.einsum('fk,bfk->bf', w32, m) + self.bias[idx].unsqueeze(0) * dp
            d_film[:, idx, 0] = df * inv
            d_film[:, idx, 1] = dp * inv
            grads[id(w)] = torch.einsum('bf,bfk->fk', f, m) * inv
            if self.wd and idx == self.c0:
                grads[id(w)] = grads[id(w)][:, 3:].contiguous()               # the reference's [feat, x]
            grads[id(b)] = (f * dp).sum(0) * inv
        L = self.L
        if fw.sigma is not None:
            grads[id(fw.sigma[0])] = (self.d_heads_w[L] * inv).reshape(fw.sigma[0].shape)
            grads[id(fw.sigma[1])] = (self.d_heads_b[L] * inv).reshape(fw.sigma[1].shape)
        if self.br:
            grads[id(fw.bridge[0])] = self.d_wv * inv
            grads[id(fw.bridge[1])] = self.d_bv * inv
        if self.res:
            # the folded maps back to their Linears, in fp64: color_layer_pre and the first colour layer's x columns from
            # the gradient of the folded [dir, v] weight g and bias gb; the density chain from d a, d c
            w, b = fw.color[0]
            g, gb = grads[id(w)].double(), grads[id(b)].double()
            wx = w.detach().double()[:, 3:]
            pw, pb = (t.detach().double() for t in fw.pre)
            grads[id(w)] = torch.cat([g[:, :3], g[:, 3:] @ pw.t() + torch.outer(gb, pb)], dim=1).float()
            grads[id(fw.pre[0])] = (wx.t() @ g[:, 3:]).float()
            grads[id(fw.pre[1])] = (wx.t() @ gb).float()
            chain = _linear_chain_grads(fw.density, (self.d_a * inv).reshape(1, 3), (self.d_c * inv).reshape(1))
            for (dw_, db_), (gw, gbb) in zip(fw.density, chain):
                grads[id(dw_)] = gw.float()
                grads[id(db_)] = gbb.float()
        n_rgb = self.spec.rgb_dim
        grads[id(fw.rgb[0])] = self.d_rgb_w[:n_rgb] * inv
        grads[id(fw.rgb[1])] = self.d_rgb_b[:n_rgb] * inv
        if self.lf:
            (hw, hb), = fw.labels
            grads[id(hw)] = self.d_heads_w[:L] * inv
            grads[id(hb)] = self.d_heads_b[:L] * inv
        elif L:
            chain = _label_chain_grads(fw.labels, self.d_heads_w[:L] * inv, self.d_heads_b[:L] * inv)
            for (w, b), (gw, gb) in zip(fw.labels, chain):
                grads[id(w)] = gw.float()
                grads[id(b)] = gb.float()
        if fw.grid is not None:
            out = torch.empty_like(fw.grid, dtype=torch.float32)
            _lib.check(_lib.lib().fenerf_grid_unpack_grad(C.byref(self.packed.desc), self.grid_grad_cl.data_ptr(), out.data_ptr(),
                                                          inv.data_ptr(), _stream(self.dev)))
            grads[id(fw.grid)] = out
        return d_film, grads


class RenderFunction(torch.autograd.Function):
    """pixels = render(film, field parameters); see the module docstring."""

    @staticmethod
    @torch.amp.custom_fwd(device_type='cuda', cast_inputs=torch.float32)
    def forward(ctx, film, call, *params):
        module, rd = call['module'], call['rd']
        st = ops.render_forward_stages(module, rd, film, call['x_lin'], call['y_lin'], call['z_lin'], call['cam2world'],
                                       call['rng_perturb'], call['rng_noise_c'], call['rng_u'], call['rng_noise_f'])
        ctx.call, ctx.stages = call, st
        ctx.save_for_backward(film, *params)
        ctx.param_ids = [id(p) for p in call['params']]
        return st['pixels']

    @staticmethod
    @torch.amp.custom_bwd(device_type='cuda')
    def backward(ctx, d_pixels):
        call, st = ctx.call, ctx.stages
        film = ctx.saved_tensors[0]
        module, rd = call['module'], call['rd']
        dev = film.device
        lib = _lib.lib()
        B, n, s = rd.batch, rd.img_h * rd.img_w, rd.num_steps
        c = st['raw_c'].shape[-1]
        hier = bool(rd.hierarchical)
        d_pixels = d_pixels.float().contiguous()
        with torch.cuda.device(dev), torch.no_grad():
            d_raw_c = torch.empty_like(st['raw_c'])
            d_raw_f = torch.empty_like(st['raw_f']) if hier else None
            noise = call['rng_noise_f'] if rd.noise_std != 0.0 else None
            if call.get('grad_rays') is not None:
                # gradient only through the chosen rays: the others were rendered under no_grad in the reference
                mask = torch.zeros(n, dtype=torch.bool, device=dev)
                mask[call['grad_rays']] = True
                d_pixels = d_pixels * mask.reshape(1, 1, rd.img_h, rd.img_w)
            _lib.check(lib.fenerf_composite_backward(
                C.byref(rd), c, st['raw_c'].data_ptr(), st['z_c'].data_ptr(), _ptr(st['raw_f']) if hier else 0,
                _ptr(st['z_f']) if hier else 0, _ptr(noise), d_pixels.data_ptr(), d_raw_c.data_ptr(), _ptr(d_raw_f),
                _stream(dev)))
            m = d_raw_c.abs().max()
            if hier:
                m = torch.maximum(m, d_raw_f.abs().max())
            scale = torch.exp2(4.0 - torch.ceil(torch.log2(m.clamp_min(1e-30)))).float().reshape(1)
            inv_scale = (1.0 / scale).float().reshape(1)
            # precision='split' renders forward on the split-precision kernel and differentiates as 'exact' does
            split = rd.precision == _lib.PRECISION['split']
            fb = _FieldBackward(module, film, scale, inv_scale, exact=split or rd.precision == _lib.PRECISION['exact'],
                                split=split, grad_split=call.get('grad_precision') == 'split')
            lock = bool(rd.lock_view_dependence)
            rays = call.get('grad_rays')
            dirs = st['dirs']

            def pick(t, last):
                # (B, n, s, last) -> (B, n' * s, last): every ray, or only the rays that carry a gradient (part_forward)
                if rays is not None:
                    t = t.index_select(1, rays)
                return t.reshape(B, -1, last)

            if rays is not None:
                dirs = dirs.index_select(1, rays).contiguous()
            if hier:
                fb.add_points(pick(st['points_f'], 3), dirs, s, lock, pick(st['raw_f'], c), pick(d_raw_f, c))
            fb.add_points(pick(st['points_c'], 3), dirs, s, lock, pick(st['raw_c'], c), pick(d_raw_c, c))
            d_film, grads = fb.finish()
        out = [d_film if ctx.needs_input_grad[0] else None, None]
        for i, pid in enumerate(ctx.param_ids):
            g = grads.get(pid) if ctx.needs_input_grad[2 + i] else None
            if g is not None:
                g = g.reshape(ctx.saved_tensors[1 + i].shape)
            out.append(g)
        return tuple(out)


class RaysRenderFunction(torch.autograd.Function):
    """pixels (B, N, C-1) = render of caller-supplied rays (fenerf_render_rays; DoubleImplicitGenerator3d.point_forward),
    differentiable w.r.t. `film` and the field parameters.  The ray tensors are inputs without gradient: the backward
    below is RenderFunction's with the ray-major compositing backward and the caller's directions."""

    @staticmethod
    @torch.amp.custom_fwd(device_type='cuda', cast_inputs=torch.float32)
    def forward(ctx, film, call, *params):
        module, rd = call['module'], call['rd']
        st = ops.render_rays_stages(module, rd, film, call['points'], call['dirs'], call['origins'], call['ray_dirs'],
                                    call['z_vals'], call['rng_noise_c'], call['rng_u'], call['rng_noise_f'])
        ctx.call, ctx.stages = call, st
        ctx.save_for_backward(film, *params)
        ctx.param_ids = [id(p) for p in call['params']]
        return st['pixels']

    @staticmethod
    @torch.amp.custom_bwd(device_type='cuda')
    def backward(ctx, d_pixels):
        call, st = ctx.call, ctx.stages
        film = ctx.saved_tensors[0]
        module, rd = call['module'], call['rd']
        dev = film.device
        B, s = rd.batch, rd.num_steps
        c = st['raw_c'].shape[-1]
        hier = bool(rd.hierarchical)
        d_pixels = d_pixels.float().contiguous()
        with torch.cuda.device(dev), torch.no_grad():
            d_raw_c = torch.empty_like(st['raw_c'])
            d_raw_f = torch.empty_like(st['raw_f']) if hier else None
            noise = call['rng_noise_f'] if rd.noise_std != 0.0 else None
            _lib.check(_lib.lib().fenerf_composite_backward_rays(
                C.byref(rd), c, st['raw_c'].data_ptr(), st['z_c'].data_ptr(), _ptr(st['raw_f']) if hier else 0,
                _ptr(st['z_f']) if hier else 0, _ptr(noise), d_pixels.data_ptr(), d_raw_c.data_ptr(), _ptr(d_raw_f),
                _stream(dev)))
            m = d_raw_c.abs().max()
            if hier:
                m = torch.maximum(m, d_raw_f.abs().max())
            scale = torch.exp2(4.0 - torch.ceil(torch.log2(m.clamp_min(1e-30)))).float().reshape(1)
            inv_scale = (1.0 / scale).float().reshape(1)
            split = rd.precision == _lib.PRECISION['split']
            fb = _FieldBackward(module, film, scale, inv_scale, exact=split or rd.precision == _lib.PRECISION['exact'],
                                split=split, grad_split=call.get('grad_precision') == 'split')
            g = st['dir_group']
            if hier:
                # the fine pass: the fine samples' own directions (per-sample), the per-ray ones, or (0, 0, -1)
                lock = bool(rd.lock_view_dependence)
                dirs_f = st['dirs_f'] if st['dirs_f'] is not None else st['dirs']
                fb.add_points(st['points_f'].reshape(B, -1, 3), dirs_f, g, lock, st['raw_f'].reshape(B, -1, c),
                              d_raw_f.reshape(B, -1, c))
            # the coarse pass keeps the caller's directions whatever lock_view_dependence says
            fb.add_points(st['points_c'].reshape(B, -1, 3), st['dirs'], g, False, st['raw_c'].reshape(B, -1, c),
                          d_raw_c.reshape(B, -1, c))
            d_film, grads = fb.finish()
        out = [d_film if ctx.needs_input_grad[0] else None, None]
        for i, pid in enumerate(ctx.param_ids):
            gr = grads.get(pid) if ctx.needs_input_grad[2 + i] else None
            if gr is not None:
                gr = gr.reshape(ctx.saved_tensors[1 + i].shape)
            out.append(gr)
        return tuple(out)


#: what a rays-in render refuses to differentiate
RAYS_GRAD_MESSAGE = ("fenerf_b200: point_forward differentiates w.r.t. the latents and the field parameters only; gradients "
                     "w.r.t. the sample points, directions, origins or depths are not built (%s requires grad): detach it")


def check_rays_no_grad(**tensors):
    """RuntimeError naming the first ray tensor that requires grad (under autograd): no gradient is silently dropped."""
    if not torch.is_grad_enabled():
        return
    for name, t in tensors.items():
        if t is not None and t.requires_grad:
            raise RuntimeError(RAYS_GRAD_MESSAGE % name)


def render_rays_with_grad(module, rd, film, points, dirs, origins, ray_dirs, z_vals, rng_noise_c, rng_u, rng_noise_f,
                          grad_precision=None):
    """Differentiable render of caller-supplied rays (rd from ops.make_rays_desc): (B, N, C-1) pixels with autograd
    edges to `film` and the field parameters.  `grad_precision` as render_with_grad."""
    check_grad_precision(module, grad_precision, rd.precision)
    check_rays_no_grad(points=points, directions=dirs, origins=origins, ray_directions=ray_dirs, z_vals=z_vals)
    params = FieldWeights(module).parameters()
    call = dict(module=module, rd=rd, points=points, dirs=dirs, origins=origins, ray_dirs=ray_dirs, z_vals=z_vals,
                rng_noise_c=rng_noise_c, rng_u=rng_u, rng_noise_f=rng_noise_f, params=params, grad_precision=grad_precision)
    return RaysRenderFunction.apply(film, call, *params)


def render_with_grad(module, rd, film, x_lin, y_lin, z_lin, cam2world, rng_perturb, rng_noise_c, rng_u, rng_noise_f,
                     grad_rays=None, grad_precision=None):
    """Differentiable render: (B, C-1, R, R) pixels with autograd edges to `film` and the field parameters.
    `grad_rays`: optional int64 ray indices -- only these rays carry the gradient (part_forward).
    `grad_precision`: None (the backward of the forward precision) or 'split' (fp32 streams, the 256-wide products on the
    split kernels of csrc/gemm_split.cu; forward precision 'split' or 'exact', the fields the split forward serves)."""
    check_grad_precision(module, grad_precision, rd.precision)
    fw = FieldWeights(module)
    params = fw.parameters()
    call = dict(module=module, rd=rd, x_lin=x_lin, y_lin=y_lin, z_lin=z_lin, cam2world=cam2world, rng_perturb=rng_perturb,
                rng_noise_c=rng_noise_c, rng_u=rng_u, rng_noise_f=rng_noise_f, params=params, grad_rays=grad_rays,
                grad_precision=grad_precision)
    return RenderFunction.apply(film, call, *params)
