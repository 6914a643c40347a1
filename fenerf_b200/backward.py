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
products (heads, the 3 / 35-wide inputs) go to the library.  ``precision='exact'`` uses fp32 library GEMMs, or, with
``grad_precision='split'``, the split kernels of csrc/gemm_split.cu on the same fp32 streams (fp16 hi / lo operands scaled
by powers of two, fp32-grade results).  One stream object per backward (_Stream) holds its weight forms
and forms these three products.  (The kernels can also fold the next layer's gate multiply
into the dA product's epilogue and produce the bias column sums from the dW kernel's staged tiles -- measured: the gate kernel's
17 ms disappear but the two GEMMs slow down by as much, both being HBM-bound; the chain below keeps the separate gate kernel.)
"""
import contextlib
import ctypes as C

import torch

from . import _lib, ops, packing

CHUNK_POINTS = 1 << 19


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


class _Stream:
    """The gradient stream of a backward: its weight forms and its three 256-wide products per FiLM layer.
      'fp16'   the default: fp16 activations, gates and dU; the products on the wgmma kernels of csrc/gemm.cu
      'exact'  precision='exact' (and 'split' renders): fp32 activations, gates and dU; the products as fp32 torch GEMMs
      'split'  grad_precision='split': the exact stream's tensors, the products on the split kernels of csrc/gemm_split.cu;
               every weight and every image's (diag(f_b) W)^T split as (hi, lo, amax), and max |dU| as dU's scale
    `film`, `bias`: the FiLM table and the biases by FiLM row; `narrow_w`: the first colour layer's fp32 weights of its
    [dir, grid features]; `rows`: the recompute's fp32 (256, 256) weights by FiLM row (None at row 0: its inputs are the
    points); `fW`: the chain products' diag(f_b) W, (B, n_film - 1, 256, 256) fp32.  (It keeps no reference to the
    _FieldBackward: no cycle, so the backward's device buffers are freed the moment it returns.)"""

    def __init__(self, kind, film, bias, narrow_w, rows, fW):
        self.kind, self.film, self.bias, self.narrow_w = kind, film, bias, narrow_w
        # element type of the activations, gates and dU, and its code in the C-ABI
        self.dt, self.dtc = (torch.float16, 0) if kind == 'fp16' else (torch.float32, 1)
        if kind == 'fp16':
            self.W = [None if w is None else w.to(torch.float16).contiguous() for w in rows]
            self.fW = fW.transpose(2, 3).to(torch.float16).contiguous()          # the NT kernel wants it transposed
            self.Wn64 = torch.zeros((256, 64), dtype=torch.float16, device=film.device)
            self.Wn64[:, :narrow_w.shape[1]] = narrow_w
            return
        self.W = [None if w is None else w.float().contiguous() for w in rows]
        self.fW = fW
        if kind == 'split':
            self.W = [None] + [ops.split_weights(w) for w in self.W[1:]]
            self.fW = ops.split_weights(fW.transpose(2, 3))

    def stash(self, z, row, b0, P, ppb, xin=None, wx=None):
        """(a, gate) of FiLM row `row` from its pre-activation z (None: zero) plus the narrow inputs xin wx^T
        (fenerf_film_forward_stash): the first layer, a bridge field's first colour layer, the exact / split recompute."""
        dev = self.film.device
        a = torch.empty((P, 256), dtype=self.dt, device=dev)
        g = torch.empty((P, 256), dtype=self.dt, device=dev)
        kx = 0 if xin is None else xin.shape[1]
        _lib.check(_lib.lib().fenerf_film_forward_stash(
            _ptr(z), self.bias[row].data_ptr(), self.film[b0, row].data_ptr(), self.film.stride(0), P, ppb,
            _ptr(xin), kx, _ptr(wx), a.data_ptr(), g.data_ptr(), self.dtc, _stream(dev)))
        return a, g

    def recompute(self, row, a_prev, b0, ppb, narrow=None):
        """(a, gate) of FiLM row `row` from the previous layer's activations.  `narrow`: the first colour layer's other
        inputs [dir, grid features]; on fp16 they ride as a fifth 64-wide k-chunk of the same kernel."""
        if self.kind == 'fp16':     # z = a W^T with the FiLM epilogue fused: z never leaves the SM
            if narrow is None:
                return ops.gemm_nt_film(a_prev, self.W[row], self.bias[row], self.film, b0, row, ppb)
            e64 = torch.zeros((a_prev.shape[0], 64), dtype=torch.float16, device=self.film.device)
            e64[:, :self.narrow_w.shape[1]] = narrow
            return ops.gemm_nt_film(a_prev, self.W[row], self.bias[row], self.film, b0, row, ppb, narrow_in=e64, narrow_w=self.Wn64)
        if self.kind == 'split' and narrow is None:
            return ops.gemm_nt_film_split(a_prev, *self.W[row], self.bias[row], self.film, b0, row, ppb)
        z = ops.gemm_nt_split(a_prev, *self.W[row]) if self.kind == 'split' else torch.mm(a_prev, self.W[row].t())
        return self.stash(z, row, b0, a_prev.shape[0], ppb, xin=narrow, wx=None if narrow is None else self.narrow_w)

    def chain(self, dU, row, b0, b1, ppb, amax):
        """dU diag(f_b) W of FiLM row `row` for each image b of the chunk: the gradient of the layer's input (P, 256)."""
        k = b1 - b0
        if self.kind == 'exact':
            return torch.bmm(dU.view(k, ppb, 256), self.fW[b0:b1, row - 1]).view(k * ppb, 256)
        out = torch.empty_like(dU)
        for i in range(k):
            rows = slice(i * ppb, (i + 1) * ppb)
            if self.kind == 'fp16':
                ops.gemm_nt(dU[rows], self.fW[b0 + i, row - 1], torch.float16, out=out[rows])
            else:
                hi, lo, w_amax = (t[b0 + i, row - 1] for t in self.fW)
                ops.gemm_nt_split(dU[rows], hi, lo, w_amax, a_amax=amax, out=out[rows])
        return out

    def weight_product(self, dU, a_in, k, ppb, amax):
        """The per-image M_b = dU_b^T a_in, (k, 256, 256) fp32."""
        if self.kind == 'fp16':
            return ops.gemm_tn(dU, a_in, k, ppb)
        if self.kind == 'split':
            return ops.gemm_tn_split(dU, a_in, k, ppb, x_amax=amax)
        return torch.bmm(dU.view(k, ppb, 256).transpose(1, 2), a_in.view(k, ppb, 256))

    def scale(self, dU):
        """max |dU| on the device for the split products; None on the other streams."""
        return ops.absmax(dU) if self.kind == 'split' else None


class _FieldBackward:
    """Accumulates the gradients of one field over any number of point sets."""

    def __init__(self, module, film, scale, inv_scale, exact=False, split=False, grad_split=False):
        # grad_split (grad_precision='split'): the fp32 streams of the exact mode, the 256-wide products on the split
        # kernels of csrc/gemm_split.cu
        if grad_split and not exact:
            raise RuntimeError(_GRAD_SPLIT_STREAMS)
        if grad_split and _grad_split_refusal(module.field_spec()):
            raise RuntimeError(_grad_split_refusal(module.field_spec()))
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
        self.T, self.c0, self.n_film = T, T + self.lf, T + self.lf + Cn
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
        # the narrow products' weights and the 256-wide weights of the gradient stream
        fw = self.fw
        self.W0 = fw.trunk[0][0].detach().float().contiguous()                    # (256, 3); grid trunk (256, G + 3)
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
        # the weights the grid features meet, (256, G): the first colour layer's, or the first layer's with the grid in
        # the trunk, whose FiLM row is then 0
        self.feat_row = 0 if self.gt else self.c0
        self.Wfeat32 = (self.W0[:, :G] if self.gt else wc0[:, 3:self.kx].contiguous()) if G else None
        if self.lf:
            self.Wlhead32 = fw.labels[0][0].detach().float().contiguous()                 # (L, 256)
        # the 256-wide weights by FiLM row (row 0 has none: its inputs are the points): trunk, label FiLM layer, colour
        wide = ([None] + [w.detach() for w, _ in fw.trunk[1:] + fw.label_film] + [wc0[:, self.kx:]]
                + [w.detach() for w, _ in fw.color[1:]])
        # the chain products dA' = dU diag(f_b) W use the same weights, except a bridge field's first colour layer: it
        # passes dU diag(f_b) W_c0[:, v] W_v (rank 3) to the trunk
        chain = list(wide)
        if self.br:
            chain[self.c0] = (self.Wc0eff[:, 3:6].double() @ self.Wv32.double()).float()
        # ... scaled per image once for every chunk: diag(f_b) W, (B, n_film - 1, 256, 256)
        fW = self.film[:, 1:, 0].unsqueeze(3) * torch.stack([w.float() for w in chain[1:]])
        self.stream = _Stream('split' if grad_split else 'exact' if exact else 'fp16', self.film, self.bias, self.Wc0x_narrow,
                              wide, fW)
        self.dt, self.dtc = self.stream.dt, self.stream.dtc       # fp16, or fp32 with precision='exact' / 'split'
        self.fWfeat = (self.film[:, self.feat_row, 0].unsqueeze(2) * self.Wfeat32).to(self.dt) if G else None    # (B, 256, G)
        # the direction-free field: TF32 rounding would be amplified like fp16's (see above); grad_split: its narrow
        # products stay fp32
        self._narrow_precision = _NoTF32 if self.wd or grad_split else contextlib.nullcontext
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
    # ray_grad: optional (B, ppb, 3) fp32 outputs 'dx' (d points, coarse pass) and 'ddir' (d direction per point), in the
    # scaled stream units (times `scale`, without input_scale); None: the backward runs exactly as without them
    def add_points(self, points, dirs, dir_group, lock_dirs, raw, d_raw, ray_grad=None):
        B, ppb, _ = points.shape

        def outs(rows, cols):
            return None if ray_grad is None else {k: (v[rows, cols] if v is not None else None) for k, v in ray_grad.items()}

        with self._narrow_precision():
            if ppb <= CHUNK_POINTS:
                k = max(1, CHUNK_POINTS // ppb)
                for b0 in range(0, B, k):
                    b1 = min(B, b0 + k)
                    self._chunk(points[b0:b1], dirs[b0:b1], dir_group, lock_dirs, raw[b0:b1], d_raw[b0:b1], b0, b1,
                                outs(slice(b0, b1), slice(None)))
                return
            step = CHUNK_POINTS // dir_group * dir_group
            for b in range(B):
                for p0 in range(0, ppb, step):
                    p1 = min(ppb, p0 + step)
                    self._chunk(points[b:b + 1, p0:p1], dirs[b:b + 1, p0 // dir_group:p1 // dir_group], dir_group, lock_dirs,
                                raw[b:b + 1, p0:p1], d_raw[b:b + 1, p0:p1], b, b + 1, outs(slice(b, b + 1), slice(p0, p1)))

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

    def _chunk(self, points, dirs, dir_group, lock_dirs, raw, d_raw, b0, b1, ray_grad=None):
        lib = _lib.lib()
        want_dx = ray_grad is not None and ray_grad.get('dx') is not None
        want_dir = ray_grad is not None and ray_grad.get('ddir') is not None
        dx_grid = dx_res = None
        dev, spec = self.dev, self.spec
        k, ppb = points.shape[0], points.shape[1]
        P = k * ppb
        T, c0 = self.T, self.c0
        stream = self.stream
        points = points.contiguous()
        dirs = dirs.contiguous()
        raw = raw.contiguous()
        d_raw = d_raw.contiguous()
        with torch.cuda.device(dev):
            st = _stream(dev)
            # ---- recompute the forward, stashing activations and gates ----
            x = (points.reshape(P, 3) * spec.input_scale).contiguous() if spec.input_scale != 1.0 else points.reshape(P, 3)
            G = spec.grid_channels
            extras = torch.empty((P, 3 + G), dtype=torch.float32, device=dev)     # [dir, feat]
            _lib.check(lib.fenerf_extras_gather(C.byref(self.packed.desc), self.packed.ptr, points.data_ptr(), dirs.data_ptr(),
                                                P, ppb, dir_group, int(bool(lock_dirs)), extras.data_ptr(), st))
            if self.gt:     # the first layer takes [feat, pos] (the reference's column order), the colour layer [dir]
                x = torch.cat([extras[:, 3:], x], dim=1).contiguous()
                extras = extras[:, :3].contiguous()
            A, Gt = [None] * self.n_film, [None] * self.n_film
            A[0], Gt[0] = stream.stash(None, 0, b0, P, ppb, xin=x, wx=self.W0)
            for l in range(1, c0):     # the trunk, then the label FiLM layer on the trunk output
                A[l], Gt[l] = stream.recompute(l, A[l - 1], b0, ppb)
            v = None
            if self.br:     # v off the trunk output (fp32), then the first colour layer on [dir, v] like a first layer
                v = _mm32(A[T - 1], self.Wv32.t().to(self.dt)) + self.bv32
                if self.res:
                    v = v + x
                extras = torch.cat([extras, v], dim=1).contiguous()
                A[c0], Gt[c0] = stream.stash(None, c0, b0, P, ppb, xin=extras, wx=self.Wc0eff)
            else:
                A[c0], Gt[c0] = stream.recompute(c0, A[T - 1], b0, ppb, narrow=extras)
            for l in range(c0 + 1, self.n_film):
                A[l], Gt[l] = stream.recompute(l, A[l - 1], b0, ppb)
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
            for idx in range(self.n_film - 1, c0 - 1, -1):
                self._gate(dA, Gt[idx], idx, b0, b1, P, ppb)                   # dA is dU now
                amax = stream.scale(dA)
                if self.br and idx == c0:
                    dv = self._bridge_back(dA, extras, v, A[T - 1], d_sigma, k, ppb, b0, b1)
                    if want_dir:
                        ray_grad['ddir'].copy_(self._narrow_grad(dA, self.Wc0eff[:, 0:3], c0, k, ppb, b0, b1))
                    if want_dx and self.res:      # v = x + res_coord_layer(a): dv (with dsigma a) reaches x
                        dx_res = dv
                else:
                    a_in = A[idx - 1] if idx > c0 else A[T - 1]
                    self.dW_b[idx][b0:b1] += stream.weight_product(dA, a_in, k, ppb, amax)
                    if idx == c0:     # the narrow inputs [dir, grid features]: their weights, the grid, d dir
                        e16 = torch.zeros((P, self.kx_pad), dtype=self.dt, device=dev)
                        e16[:, :self.kx] = extras
                        self.dWx_b[b0:b1] += _bmm32(dA.view(k, ppb, 256).transpose(1, 2), e16.view(k, ppb, self.kx_pad))
                        if G and not self.gt:
                            d_feat = self._grid_grad(dA, points, k, ppb, b0, b1)
                            if want_dx:
                                dx_grid = self._coord_grad(d_feat, points, P)
                        if want_dir:
                            ray_grad['ddir'].copy_(self._narrow_grad(dA, self.Wc0x_narrow[:, 0:3], c0, k, ppb, b0, b1))
                dA = stream.chain(dA, idx, b0, b1, ppb, amax)
                A[idx], Gt[idx] = None, None
            # ---- trunk: colour-branch gradient + sigma / label heads ----
            dA += torch.mm(dH.float(), self.Wheads32)
            if self.lf:     # label branch: d logits W_head -> gate -> M_b, colsum of row T; dU diag(f) W_label joins the trunk's dA
                # (P, 256), formed in fp32: an fp16 product's reduction order depends on the chunk's row count
                dAl = torch.mm(dH[:, :self.L].float(), self.Wlhead32).to(self.dt)
                self._gate(dAl, Gt[T], T, b0, b1, P, ppb)
                amax = stream.scale(dAl)
                self.dW_b[T][b0:b1] += stream.weight_product(dAl, A[T - 1], k, ppb, amax)
                dA += stream.chain(dAl, T, b0, b1, ppb, amax)
                A[T], Gt[T] = None, None
            for l in range(T - 1, 0, -1):
                self._gate(dA, Gt[l], l, b0, b1, P, ppb)
                amax = stream.scale(dA)
                self.dW_b[l][b0:b1] += stream.weight_product(dA, A[l - 1], k, ppb, amax)
                dA = stream.chain(dA, l, b0, b1, ppb, amax)
                A[l], Gt[l] = None, None
            self._gate(dA, Gt[0], 0, b0, b1, P, ppb)
            if self.gt:
                d_feat = self._grid_grad(dA, points, k, ppb, b0, b1)
                if want_dx:
                    dx_grid = self._coord_grad(d_feat, points, P)
            if want_dx:     # x = points * input_scale: the first layer's position columns, the grid term, RES's dv
                dx = self._narrow_grad(dA, self.W0[:, self.k0 - 3:self.k0], 0, k, ppb, b0, b1)
                if dx_grid is not None:
                    dx += dx_grid.view(k, ppb, 3)
                if dx_res is not None:
                    dx += dx_res.view(k, ppb, 3)
                ray_grad['dx'].copy_(dx)
            x16 = torch.zeros((P, self.k0_pad), dtype=self.dt, device=dev)
            x16[:, :self.k0] = x
            self.dW_b[0][b0:b1] += _bmm32(dA.view(k, ppb, 256).transpose(1, 2), x16.view(k, ppb, self.k0_pad))

    def _bridge_back(self, dU, extras, v, a_trunk, d_sigma, k, ppb, b0, b1):
        """First colour layer of a bridge field on [dir, v]: its narrow weight gradient, dv = dU diag(f) W_c0[:, v]
        (+ dsigma a for RES) and v's own gradients, in fp32 (3 columns).  The trunk's share dv W_v goes through the chain
        product and the sigma head instead (see the module docstring)."""
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
        return dv

    def _narrow_grad(self, dU, w, row, k, ppb, b0, b1):
        """dU diag(f_b) w of FiLM row `row` for a narrow slice w (256, 3) of the layer's input columns: the gradient of
        those inputs, (k, ppb, 3) fp32 (ray_grad)."""
        with _NoTF32():
            return torch.bmm(dU.view(k, ppb, 256).float(), self.film[b0:b1, row, 0].unsqueeze(2) * w)

    def _coord_grad(self, d_feat, points, P):
        """The grid term of the sample points' gradient, (P, 3) fp32 w.r.t. the box-warped coordinate (ray_grad)."""
        out = torch.empty((P, 3), dtype=torch.float32, device=self.dev)
        _lib.check(_lib.lib().fenerf_grid_coord_grad(C.byref(self.packed.desc), self.packed.ptr, points.data_ptr(),
                                                     d_feat.data_ptr(), d_feat.shape[1], P, out.data_ptr(),
                                                     1 if d_feat.dtype == torch.float32 else 0, _stream(self.dev)))
        return out

    def _grid_grad(self, dU, points, k, ppb, b0, b1):
        """d features = dU diag(f_b) W_feat, (P, G), of the layer the grid feeds, scattered into the grid accumulator."""
        P = k * ppb
        d_feat = torch.bmm(dU.view(k, ppb, 256), self.fWfeat[b0:b1]).view(P, -1).contiguous()
        if self.det:     # 64-bit fixed point at a scale taken from this point set's max |d feat|, integer atomics
            ws = self.grid_det_ws
            _lib.check(_lib.lib().fenerf_grid_scatter_add_det(C.byref(self.packed.desc), points.data_ptr(), d_feat.data_ptr(),
                                                              d_feat.shape[1], P, ws.data_ptr(), ws.numel(),
                                                              self.grid_grad_cl.data_ptr(), self.dtc, _stream(self.dev)))
            return d_feat
        _lib.check(_lib.lib().fenerf_grid_scatter_add(C.byref(self.packed.desc), points.data_ptr(), d_feat.data_ptr(),
                                                      d_feat.shape[1], P, self.grid_grad_cl.data_ptr(), self.dtc,
                                                      _stream(self.dev)))
        return d_feat

    # ---- after every point set: fold the per-image accumulators into parameter / FiLM gradients ----
    def finish(self):
        with self._narrow_precision():
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


def _field_backward(call, film, d_raw_c, d_raw_f):
    """The _FieldBackward of a render: its precision and grad_precision, the fp16 stream's scale a power of two taken from
    max |d raw| on the device (no host sync)."""
    module, rd = call['module'], call['rd']
    m = d_raw_c.abs().max()
    if d_raw_f is not None:
        m = torch.maximum(m, d_raw_f.abs().max())
    scale = torch.exp2(4.0 - torch.ceil(torch.log2(m.clamp_min(1e-30)))).float().reshape(1)
    inv_scale = (1.0 / scale).float().reshape(1)
    # precision='split' renders forward on the split-precision kernel and differentiates as 'exact' does
    split = rd.precision == _lib.PRECISION['split']
    return _FieldBackward(module, film, scale, inv_scale, exact=split or rd.precision == _lib.PRECISION['exact'], split=split,
                          grad_split=call.get('grad_precision') == 'split')


#: the ray set-up inputs of a camera render, and the ray tensors of a rays-in render in the order RenderFunction takes them
#: with ray_grad
CAMERA_INPUTS = ("x_lin", "y_lin", "z_lin", "cam2world", "rng_perturb")
RAY_INPUTS = ("points", "dirs", "origins", "ray_dirs", "z_vals")


class RenderFunction(torch.autograd.Function):
    """pixels = render(film, field parameters); see the module docstring.  One node for both renders:
      camera   (call from render_with_grad) fenerf_render_forward, NCHW pixels.  A cam2world that requires grad follows the
               parameters as an input and gets the gradient of the coarse sample points R p_cam + T
               and of the ray directions R d_cam of both passes (fenerf_cam2world_grad); the fine points, the depths and
               the origins carry none, as in the reference.
      rays-in  (call from render_rays_with_grad) fenerf_render_rays, (B, N, C-1) ray-major pixels
               (DoubleImplicitGenerator3d.point_forward).  With ray_grad the ray tensors (RAY_INPUTS) follow the
               parameters as inputs and get the reference's gradients: the coarse points, the directions (both passes;
               the fine samples' through their draw slots), the depths without hierarchical sampling, and None for the
               per-ray origins and directions.
    The two differ in where the rays come from, the compositing backward of their pixel layout, which passes
    lock_view_dependence locks and where the ray gradients go; the rest of the backward is one path."""

    @staticmethod
    @torch.amp.custom_fwd(device_type='cuda', cast_inputs=torch.float32)
    def forward(ctx, film, call, *inputs):
        module, rd = call['module'], call['rd']
        n_params = len(call['params'])
        extra = inputs[n_params:]           # the cam2world that requires grad, or the ray tensors (ray_grad)
        draws = (call['rng_noise_c'], call['rng_u'], call['rng_noise_f'])
        if 'cam2world' in call:
            st = ops.render_forward_stages(module, rd, film, *(call[k] for k in CAMERA_INPUTS), *draws)
        else:
            # the fine samples' draw slots: only for a backward w.r.t. the directions
            slots = bool(extra) and ctx.needs_input_grad[2 + n_params + 1]
            st = ops.render_rays_stages(module, rd, film, *(extra or (call[k] for k in RAY_INPUTS)), *draws, slots=slots)
        ctx.call, ctx.stages = call, st
        ctx.save_for_backward(film, *inputs[:n_params])
        ctx.param_ids = [id(p) for p in call['params']]
        ctx.extra_meta = [(t.shape, t.dtype) if t is not None else None for t in extra]
        return st['pixels']

    @staticmethod
    @torch.amp.custom_bwd(device_type='cuda')
    def backward(ctx, d_pixels):
        call, st = ctx.call, ctx.stages
        film = ctx.saved_tensors[0]
        rd = call['rd']
        dev = film.device
        lib = _lib.lib()
        camera = 'cam2world' in call
        B, n, s = rd.batch, rd.img_h * rd.img_w, rd.num_steps
        c = st['raw_c'].shape[-1]
        hier = bool(rd.hierarchical)
        n_params = len(ctx.param_ids)
        need = ctx.needs_input_grad[2 + n_params:] + (False,) * len(RAY_INPUTS)     # (inputs the call lacks want none)
        spec = call['module'].field_spec()
        rays = call.get('grad_rays')
        # the consumer of the ray gradients: d cam2world reads d points and d directions; a rays-in render's caller takes
        # each ray tensor that requires grad (the direction-free field never reads directions; the depths get a gradient
        # only without hierarchical sampling)
        want_dx = need[0]
        want_dirs = need[0 if camera else 1] and not spec.wo_dir
        want_z = not camera and need[4] and not hier
        # lock_view_dependence locks both passes of a camera render, only the fine pass of a rays-in render: the coarse
        # pass keeps the caller's directions whatever it says (generators.py:810)
        lock_f = bool(rd.lock_view_dependence)
        lock_c = lock_f and camera
        d_pixels = d_pixels.float().contiguous()
        with torch.cuda.device(dev), torch.no_grad():
            d_raw_c = torch.empty_like(st['raw_c'])
            d_raw_f = torch.empty_like(st['raw_f']) if hier else None
            noise = call['rng_noise_f'] if rd.noise_std != 0.0 else None
            if rays is not None:
                # gradient only through the chosen rays: the others were rendered under no_grad in the reference
                mask = torch.zeros(n, dtype=torch.bool, device=dev)
                mask[rays] = True
                d_pixels = d_pixels * mask.reshape(1, 1, rd.img_h, rd.img_w)
            d_z = None
            if want_z:     # the same d raw, and the depth gradient beside it
                d_z = torch.empty_like(st['z_c'])
                _lib.check(lib.fenerf_composite_backward_rays_dz(
                    C.byref(rd), c, st['raw_c'].data_ptr(), st['z_c'].data_ptr(), _ptr(noise), d_pixels.data_ptr(),
                    d_raw_c.data_ptr(), d_z.data_ptr(), _stream(dev)))
            else:
                _lib.check((lib.fenerf_composite_backward if camera else lib.fenerf_composite_backward_rays)(
                    C.byref(rd), c, st['raw_c'].data_ptr(), st['z_c'].data_ptr(), _ptr(st['raw_f']), _ptr(st['z_f']),
                    _ptr(noise), d_pixels.data_ptr(), d_raw_c.data_ptr(), _ptr(d_raw_f), _stream(dev)))
            fb = _field_backward(call, film, d_raw_c, d_raw_f)

            def pick(t, last):
                # (B, n, s, last) -> (B, n' * s, last): every ray, or only the rays that carry a gradient (part_forward)
                if rays is not None:
                    t = t.index_select(1, rays)
                return t.reshape(B, -1, last)

            dirs_c = st['dirs'] if rays is None else st['dirs'].index_select(1, rays).contiguous()
            # the fine pass: a rays-in render's fine samples' own directions (per-sample), else the coarse pass's
            dirs_f = st['dirs_f'] if st['dirs_f'] is not None else dirs_c
            g = st['dir_group']

            def buf():
                return torch.zeros((B, n * s, 3), dtype=torch.float32, device=dev)

            # d points of the coarse pass, d direction per point of each pass that reads unlocked directions
            dx = buf() if want_dx else None
            dir_c = buf() if want_dirs and not lock_c else None
            dir_f = buf() if want_dirs and hier and not lock_f else None
            if hier:
                fb.add_points(pick(st['points_f'], 3), dirs_f, g, lock_f, pick(st['raw_f'], c), pick(d_raw_f, c),
                              ray_grad=dict(ddir=dir_f) if dir_f is not None else None)
            fb.add_points(pick(st['points_c'], 3), dirs_c, g, lock_c, pick(st['raw_c'], c), pick(d_raw_c, c),
                          ray_grad=dict(dx=dx, ddir=dir_c) if (dx is not None or dir_c is not None) else None)
            d_film, grads = fb.finish()
            d_dirs = None
            if dir_c is not None:     # the directions' gradients per ray (dir_group S) or per sample
                d_dirs = torch.empty((B * n * s // g, 3), dtype=torch.float32, device=dev)
                _lib.check(lib.fenerf_ray_dir_grad(B * n, s, g, dir_c.data_ptr(), _ptr(dir_f),
                                                   _ptr(st['slots_f']) if dir_f is not None else 0,
                                                   fb.inv_scale.data_ptr(), d_dirs.data_ptr(), _stream(dev)))
            if camera:
                extra = [_cam2world_grad(call, fb, dx, d_dirs) if want_dx else None]
            else:
                extra = [dx * fb.inv_scale * spec.input_scale if dx is not None else None, d_dirs, None, None, d_z]
            if call.get('grad_reduce') is not None:
                call['grad_reduce']([d_film] + list(grads.values()) + [extra[0] if camera else None])
        out = [d_film if ctx.needs_input_grad[0] else None, None]
        for i, pid in enumerate(ctx.param_ids):
            gr = grads.get(pid) if ctx.needs_input_grad[2 + i] else None
            out.append(gr.reshape(ctx.saved_tensors[1 + i].shape) if gr is not None else None)
        for gr, meta, want in zip(extra, ctx.extra_meta, need):
            out.append(gr.reshape(meta[0]).to(meta[1]) if gr is not None and want else None)
        return tuple(out)


def _cam2world_grad(call, fb, dx, d_dirs):
    """d cam2world (B, 4, 4) of a camera render from the coarse pass's d points `dx` (scaled stream units) and the
    directions' per-ray gradients d_dirs (fenerf_ray_dir_grad; None: no direction is differentiated):
    fenerf_cam2world_grad, which recomputes the camera-space samples."""
    rd, dev = call['rd'], fb.dev
    lib = _lib.lib()
    ws = torch.empty(lib.fenerf_cam2world_grad_workspace_bytes(C.byref(rd)), dtype=torch.uint8, device=dev)
    d_c2w = torch.empty((rd.batch, 4, 4), dtype=torch.float32, device=dev)
    _lib.check(lib.fenerf_cam2world_grad(
        C.byref(rd), call['x_lin'].data_ptr(), call['y_lin'].data_ptr(), call['z_lin'].data_ptr(),
        call['rng_perturb'].data_ptr(), dx.data_ptr(), _ptr(d_dirs), fb.inv_scale.data_ptr(), fb.spec.input_scale,
        ws.data_ptr(), ws.numel(), d_c2w.data_ptr(), _stream(dev)))
    return d_c2w


#: what a rays-in render refuses to differentiate
RAYS_GRAD_MESSAGE = ("fenerf_b200: point_forward differentiates w.r.t. the latents and the field parameters only; gradients "
                     "w.r.t. the sample points, directions, origins or depths are not built (%s requires grad): detach it, "
                     "or pass ray_grad=True")


def check_rays_no_grad(**tensors):
    """RuntimeError naming the first ray tensor that requires grad (under autograd): no gradient is silently dropped."""
    if not torch.is_grad_enabled():
        return
    for name, t in tensors.items():
        if t is not None and t.requires_grad:
            raise RuntimeError(RAYS_GRAD_MESSAGE % name)


def render_rays_with_grad(module, rd, film, points, dirs, origins, ray_dirs, z_vals, rng_noise_c, rng_u, rng_noise_f,
                          grad_precision=None, ray_grad=False):
    """Differentiable render of caller-supplied rays (rd from ops.make_rays_desc): (B, N, C-1) pixels with autograd
    edges to `film` and the field parameters.  `grad_precision` as render_with_grad.  ray_grad=True: also to the ray
    tensors (RenderFunction); without it a ray tensor that requires grad is refused."""
    check_grad_precision(module, grad_precision, rd.precision)
    if not ray_grad:
        check_rays_no_grad(points=points, directions=dirs, origins=origins, ray_directions=ray_dirs, z_vals=z_vals)
    params = FieldWeights(module).parameters()
    call = dict(module=module, rd=rd, points=points, dirs=dirs, origins=origins, ray_dirs=ray_dirs, z_vals=z_vals,
                rng_noise_c=rng_noise_c, rng_u=rng_u, rng_noise_f=rng_noise_f, params=params, grad_precision=grad_precision)
    rays = (points, dirs, origins, ray_dirs, z_vals) if ray_grad else ()
    return RenderFunction.apply(film, call, *params, *rays)


def render_with_grad(module, rd, film, x_lin, y_lin, z_lin, cam2world, rng_perturb, rng_noise_c, rng_u, rng_noise_f,
                     grad_rays=None, grad_precision=None, grad_reduce=None):
    """Differentiable render: (B, C-1, R, R) pixels with autograd edges to `film` and the field parameters.
    `grad_rays`: optional int64 ray indices -- only these rays carry the gradient (part_forward).
    `grad_precision`: None (the backward of the forward precision) or 'split' (fp32 streams, the 256-wide products on the
    split kernels of csrc/gemm_split.cu; forward precision 'split' or 'exact', the fields the split forward serves).
    `grad_reduce`: optional callable given [d film, every parameter gradient, d cam2world or None] before they leave the
    backward; it may modify them in place (a ray-sharded render sums them over its ranks there, dist.RayShard.reduce).
    A `cam2world` that requires grad (a pose input of forward_with_frequencies that does) gets its gradient."""
    check_grad_precision(module, grad_precision, rd.precision)
    params = FieldWeights(module).parameters()
    pose_grad = torch.is_grad_enabled() and cam2world.requires_grad
    if pose_grad and grad_rays is not None:
        raise ValueError("fenerf_b200: the pose gradient is not built for ray subsets (grad_rays)")
    call = dict(module=module, rd=rd, x_lin=x_lin, y_lin=y_lin, z_lin=z_lin, cam2world=cam2world.detach(),
                rng_perturb=rng_perturb, rng_noise_c=rng_noise_c, rng_u=rng_u, rng_noise_f=rng_noise_f, params=params,
                grad_rays=grad_rays, grad_precision=grad_precision, grad_reduce=grad_reduce)
    return RenderFunction.apply(film, call, *params, *((cam2world,) if pose_grad else ()))
