"""Host-side mirror of the reference's FiLM-SIREN point networks (siren/siren.py).

Only the module *interface* is kept from the reference -- class names, constructor arguments,
attribute names, parameter registration order (EMA ``copy_to`` is positional), state-dict keys and
the init RNG consumption -- so that checkpoints pickled as ``siren.siren.<Class>`` load and the
reference's callers run unchanged.  The per-point arithmetic is not here: it is the sm_90a CUDA
kernel behind ``fenerf_siren_points`` (include/fenerf_b200.h).  Each network describes itself to
the kernel through a small layer table (:class:`FieldSpec`), which is how further reference variants
can be added without new kernels (SURVEY.md section 8f-4).

Reference interfaces mirrored (file:line in the reference tree):
  FiLMLayer                                   siren/siren.py:113-123
  CustomMappingNetwork                        siren/siren.py:82-102
  frequency_init / first-layer inits          siren/siren.py:45-49, 104-110, 333-338
  TALLSIREN                                   siren/siren.py:126-178
  UniformBoxWarp                              siren/siren.py:181-187
  sample_from_3dgrid                          siren/siren.py:314-330
  SPATIALSIRENBASELINE                        siren/siren.py:189-244
  EmbeddingPiGAN256                           siren/siren.py:341-410
  SPATIALSIRENSEMANTIC                        siren/siren.py:597-671
  SPATIALSIRENBASELINESEMANTIC                siren/siren.py:674-744
  SPATIALSIRENDISENTANGLE                     siren/siren.py:747-813
  SPATIALSIRENAUGDISENTANGLE                  siren/siren.py:904-979
  RESSIRENDISENTANGLE                         siren/siren.py:982-1082
  SPATIALSIRENSEMANTICDISENTANGLE             siren/siren.py:1085-1161
  SIRENBASELINESEMANTICDISENTANGLE            siren/siren.py:1163-1229
  TextureEmbeddingPiGAN128SEMANTICDISENTANGLE siren/siren.py:1451-1530
  ...256SEMANTICDISENTANGLE / ..._DIM_96      siren/siren.py:1533-1546
  TextureEmbeddingPiGAN128SEMANTICDISENTANGLE_WO_DIR / ...256..._WO_DIR_DIM_96   siren/siren.py:1549-1640, 1817-1822
"""
import math
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

HIDDEN = 256  # the kernels are specialised for 256-wide FiLM layers


# --------------------------------------------------------------------------------------------
# initialisers (same distributions and the same RNG consumption as the reference)
# --------------------------------------------------------------------------------------------
def _uniform_weight(bound_of_fan_in):
    def init(m):
        if isinstance(m, nn.Linear):
            with torch.no_grad():
                b = bound_of_fan_in(m.weight.size(-1))
                m.weight.uniform_(-b, b)
    return init


def frequency_init(freq):
    """U(+-sqrt(6/fan_in)/freq) on every nn.Linear weight (siren/siren.py:104-110)."""
    return _uniform_weight(lambda fan_in: math.sqrt(6 / fan_in) / freq)


#: U(+-1/fan_in) first-layer init (siren/siren.py:45-49); fan_in is 3 for every network here,
#: which also covers ``modified_first_sine_init`` (siren/siren.py:333-338, hard-coded 3).
first_layer_film_sine_init = _uniform_weight(lambda fan_in: 1 / fan_in)
modified_first_sine_init = _uniform_weight(lambda fan_in: 1 / 3)


def kaiming_leaky_init(m):
    if m.__class__.__name__.find('Linear') != -1:
        torch.nn.init.kaiming_normal_(m.weight, a=0.2, mode='fan_in', nonlinearity='leaky_relu')


# --------------------------------------------------------------------------------------------
# building blocks
# --------------------------------------------------------------------------------------------
class FiLMLayer(nn.Module):
    """sin(freq * (x W^T + b) + phase); the state-dict key of the Linear is ``layer``.

    ``forward`` exists for the differentiable torch path only (autograd callers, section 8f-1);
    the render path never calls it.
    """

    def __init__(self, input_dim, hidden_dim):
        super().__init__()
        self.layer = nn.Linear(input_dim, hidden_dim)

    def forward(self, x, freq, phase_shift):
        x = self.layer(x)
        if x.shape[1] != freq.shape[1]:
            freq = freq.unsqueeze(1).expand_as(x)
            phase_shift = phase_shift.unsqueeze(1).expand_as(x)
        return torch.sin(freq * x + phase_shift)


class CustomMappingNetwork(nn.Module):
    """z -> (frequencies, phase_shifts): Linear + LeakyReLU(0.2) x (1 + n_blocks), then Linear.

    Stays in PyTorch/cuBLAS (SURVEY.md section 8 row a7: ~0 % of the time).
    """

    def __init__(self, z_dim, map_hidden_dim, map_output_dim, n_blocks=3):
        super().__init__()
        dims = [z_dim] + [map_hidden_dim] * (n_blocks + 1)
        mods = []
        for d_in, d_out in zip(dims[:-1], dims[1:]):
            mods += [nn.Linear(d_in, d_out), nn.LeakyReLU(0.2, inplace=True)]
        mods.append(nn.Linear(map_hidden_dim, map_output_dim))
        self.network = nn.Sequential(*mods)
        self.network.apply(kaiming_leaky_init)
        with torch.no_grad():
            self.network[-1].weight *= 0.25

    def forward(self, z):
        out = self.network(z)
        half = out.shape[-1] // 2
        return out[..., :half], out[..., half:]


class UniformBoxWarp(nn.Module):
    def __init__(self, sidelength):
        super().__init__()
        self.scale_factor = 2 / sidelength

    def forward(self, coordinates):
        return coordinates * self.scale_factor


def sample_from_3dgrid(coordinates, grid):
    """Trilinear lookup, align_corners=True, zero padding (siren/siren.py:314-330).

    Torch formulation for the autograd path; the render path uses the channels-last gather in
    csrc/siren_common.cuh.
    """
    coordinates = coordinates.float()
    grid = grid.float()
    bsz, n_coords, n_dims = coordinates.shape
    feats = torch.nn.functional.grid_sample(
        grid.expand(bsz, -1, -1, -1, -1), coordinates.reshape(bsz, 1, 1, -1, n_dims),
        mode='bilinear', padding_mode='zeros', align_corners=True)
    n, c, h, w, d = feats.shape
    return feats.permute(0, 4, 3, 2, 1).reshape(n, h * w * d, c)


# --------------------------------------------------------------------------------------------
# kernel-facing description of a point network
# --------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class FieldSpec:
    """What the CUDA point-network kernels need to know about a FiLM-SIREN field.

    trunk_layers   FiLM layers on the position (first is 3 -> 256, rest 256 -> 256)
    color_layers   FiLM layers of the colour branch; the first consumes
                   cat[ray_dir(3), grid_feat(grid_channels), trunk_out(256)]
    label_dim      semantic logits (0 = none); the reference's activation-free Linear chain
                   (siren/siren.py:1486-1490) is pre-multiplied into one 256 -> label_dim map
    label_film     the label head is a FiLM layer on the trunk output followed by one Linear
                   (siren/siren.py:663-665); its FiLM row sits between the trunk's and the colour branch's
    grid_channels  feature-grid channels (0 = no grid)
    input_scale    UniformBoxWarp factor applied to the position before the trunk and the grid
    feature_head   the colour head is Linear(256 -> 64) without the sigmoid: 64 features for a neural renderer
                   (siren/siren.py:300-301, 1365-1366)
    grid_trunk     the grid features feed the first trunk layer, cat[feat, pos] -> 256, and not the colour branch
                   (siren/siren.py:396-398)
    bridge         the colour branch reads cat[ray_dir(3), v(3)], v = Linear(256 -> 3)(trunk output), not the trunk's 256
                   activations (siren/siren.py:965-967)
    bridge_res     with bridge: v = warped position + Linear(256 -> 3)(trunk output), the density is a chain of four
                   Linears on v and the first colour layer reads cat[ray_dir, Linear(3 -> 256)(v)] (siren/siren.py:1072-1076)
    wo_dir         the first colour layer reads cat[grid_feat, trunk_out(256)], no ray direction, and carries the U(+-1/3)
                   init (siren/siren.py:1606, 1626), which amplifies the fp16 trunk's error: the colours come from the exact
                   and the split-precision kernels only (the density alone runs in any precision)
    out_dim        label_dim + 3 (rgb; 64 features with feature_head) + 1 (sigma); channel order [labels, rgb, sigma]
    """
    trunk_layers: int
    color_layers: int
    label_dim: int
    grid_channels: int
    grid_res: int
    input_scale: float
    out_dim: int
    double_latent: bool
    label_film: bool = False
    feature_head: bool = False
    grid_trunk: bool = False
    bridge: bool = False
    bridge_res: bool = False
    wo_dir: bool = False

    @property
    def rgb_dim(self):
        return 64 if self.feature_head else 3


def _fused_mapping_ok(net, z):
    """The two-launch mapping kernels serve no_grad callers on CUDA with the reference's 256-wide, 3-block network."""
    if torch.is_grad_enabled() or not z.is_cuda or z.dtype != torch.float32:
        return False
    lin = [m for m in net.network if isinstance(m, nn.Linear)]
    return (len(lin) == 5 and lin[0].out_features == 256 and lin[0].in_features % 4 == 0 and lin[0].in_features <= 512
            and lin[-1].out_features % 512 == 0)


class _FieldBase(nn.Module):
    """Shared host logic: FiLM table assembly, weight packing cache, dispatch to the C-ABI."""

    hidden_dim = HIDDEN

    def field_spec(self) -> FieldSpec:  # pragma: no cover - overridden
        raise NotImplementedError

    # -- packed-weight cache -------------------------------------------------------------
    def _field_parameters(self):
        """The parameters the kernels consume (everything but the mapping networks, which stay in PyTorch)."""
        plist = self.__dict__.get('_field_plist')
        if plist is None or plist[0] != len(self._parameters) + sum(1 for _ in self.children()):
            ps = [p for n, p in self.named_parameters() if 'mapping_network' not in n]
            plist = (len(self._parameters) + sum(1 for _ in self.children()), ps)
            self.__dict__['_field_plist'] = plist
        return plist[1]

    def _weights_version(self):
        return tuple((p.data_ptr(), p._version) for p in self._field_parameters())

    def packed(self, verify=False, split=False):
        """Kernel-layout weights.  Repacked when a parameter's (storage, version) changed -- what optimizer
        steps and in-place torch ops bump.  Writes through ``param.data`` (torch_ema ``copy_to`` / ``restore``,
        train_double_latent_semantic.py:464-522) bump nothing: ``verify=True`` compares a device-side
        fingerprint of the raw parameters with the one taken at pack time (one kernel + a 16-byte read-back,
        so a host sync) -- the generators pass it from ``staged_forward*``, the methods the reference renders
        EMA weights through, whose outputs go to the CPU anyway.  :meth:`invalidate_packed` forces a repack.
        ``split=True``: the pack precision='split' reads, which also holds the fp16 low parts of the weight images
        (FENERF_FIELD_SPLIT_IMAGES); cached beside the other under the same rules and made on first use only.
        """
        from .. import packing
        key = '_packed_split_cache' if split else '_packed_cache'
        ver = self._weights_version()
        cache = self.__dict__.get(key)
        if cache is not None and cache[0] == ver and verify:
            fp = packing.fingerprint(self)
            if cache[1].fingerprint is None:
                # first verified use of this pack: nothing to compare with yet; a pack made by this very call
                # chain is fresh, one made by an earlier non-verified call may already be stale -> repack once
                cache = None
            elif cache[1].fingerprint != fp:
                cache = None
        if cache is None or cache[0] != ver:
            cache = (ver, packing.pack_field(self, split))
            if verify:
                cache[1].fingerprint = packing.fingerprint(self)
            self.__dict__[key] = cache
        cache[1].wait_ready()
        return cache[1]

    def invalidate_packed(self):
        """Drop the kernel-layout copy of the weights (next render repacks)."""
        self.__dict__.pop('_packed_cache', None)
        self.__dict__.pop('_packed_split_cache', None)

    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop('_packed_cache', None)  # never pickle device buffers derived from the weights
        state.pop('_packed_split_cache', None)
        state.pop('_field_plist', None)
        return state

    # -- the point-network entry the reference's callers use --------------------------------
    def _render_points(self, points, film, ray_directions):
        from .. import ops
        return ops.siren_points(self, points, film, ray_directions)

    def density(self, points, film, precision=None):
        """(B,P,3) points, (B,L,2,256) FiLM table (see film_table) -> (B,P,1) density only: what the shape
        extraction keeps of forward_with_frequencies_phase_shifts (extract_double_semantic_shapes.py:59-62),
        without evaluating the colour / label branches."""
        from .. import ops
        return ops.siren_sigma(self, points, film, precision)


class TALLSIREN(_FieldBase):
    """pi-GAN's primary SIREN: 8 FiLM + sigma head + 1 colour FiLM + sigmoid rgb (model A)."""

    def __init__(self, input_dim=2, z_dim=100, hidden_dim=256, output_dim=1, device=None):
        super().__init__()
        self.device = device
        self.input_dim = input_dim
        self.z_dim = z_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim

        widths = [input_dim] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        self.color_layer_sine = FiLMLayer(hidden_dim + 3, hidden_dim)
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3), nn.Sigmoid())
        self.mapping_network = CustomMappingNetwork(z_dim, 256, (len(self.network) + 1) * hidden_dim * 2)

        for part in (self.network, self.final_layer, self.color_layer_sine, self.color_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(first_layer_film_sine_init)

    def field_spec(self):
        return FieldSpec(trunk_layers=len(self.network), color_layers=1, label_dim=0, grid_channels=0,
                         grid_res=0, input_scale=1.0, out_dim=4, double_latent=False)

    def film_rows(self):
        """FiLM layers of the table: the trunk's and the colour layer's."""
        return len(self.network) + 1

    def film_table(self, frequencies, phase_shifts):
        """(B, L*256) raw mapping outputs -> (B, L, 2, 256) [15 f + 30, phase] (siren.py:165)."""
        b = frequencies.shape[0]
        f = (frequencies * 15 + 30).reshape(b, -1, self.hidden_dim)
        p = phase_shifts.reshape(b, -1, self.hidden_dim)
        return torch.stack([f, p], dim=2).float().contiguous()

    def film_from_latents(self, z, psi=1.0, avg=None):
        """z -> FiLM table.  Under no_grad on a CUDA device: the fused mapping kernels (fenerf_mapping_film, two
        launches); otherwise the PyTorch modules, so that autograd reaches the mapping network and the latent.
        `avg` = (avg_frequencies, avg_phase_shifts) enables the psi truncation of staged_forward."""
        from .. import ops
        n = self.film_rows()
        if _fused_mapping_ok(self.mapping_network, z):
            film = torch.empty((z.shape[0], n, 2, self.hidden_dim), dtype=torch.float32, device=z.device)
            return ops.mapping_film(self.mapping_network, z, film, 0, n, avg=avg, psi=psi)
        frequencies, phase_shifts = self.mapping_network(z)
        if avg is not None:
            frequencies = avg[0] + psi * (frequencies - avg[0])
            phase_shifts = avg[1] + psi * (phase_shifts - avg[1])
        return self.film_table(frequencies, phase_shifts)

    def forward(self, input, z, ray_directions, **kwargs):
        frequencies, phase_shifts = self.mapping_network(z)
        return self.forward_with_frequencies_phase_shifts(input, frequencies, phase_shifts, ray_directions, **kwargs)

    def forward_with_frequencies_phase_shifts(self, input, frequencies, phase_shifts, ray_directions, **kwargs):
        return self._render_points(input, self.film_table(frequencies, phase_shifts), ray_directions)


class SPATIALSIRENBASELINE(TALLSIREN):
    """TALLSIREN plus a UniformBoxWarp(0.24) on the input points (siren/siren.py:189-244); the network of the
    `CelebA` curriculum (curriculums.py:66)."""

    def __init__(self, input_dim=2, z_dim=100, hidden_dim=256, output_dim=1, device=None):
        nn.Module.__init__(self)
        self.device = device
        self.input_dim = input_dim
        self.z_dim = z_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        self.color_layer_sine = FiLMLayer(hidden_dim + 3, hidden_dim)
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3))
        self.mapping_network = CustomMappingNetwork(z_dim, 256, (len(self.network) + 1) * hidden_dim * 2)

        for part in (self.network, self.final_layer, self.color_layer_sine, self.color_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(first_layer_film_sine_init)
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        return FieldSpec(trunk_layers=len(self.network), color_layers=1, label_dim=0, grid_channels=0,
                         grid_res=0, input_scale=float(self.gridwarper.scale_factor), out_dim=4, double_latent=False)


class SPATIALSIRENBASELINESEMANTIC(TALLSIREN):
    """SPATIALSIRENBASELINE plus a two-Linear semantic head with a fixed 19 labels (siren/siren.py:674-744):
    output channels [labels (19), rgb (3), sigma (1)] whatever `output_dim` says."""

    def __init__(self, input_dim=2, z_dim=100, hidden_dim=256, output_dim=1, device=None):
        nn.Module.__init__(self)
        self.device = device
        self.input_dim = input_dim
        self.z_dim = z_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        self.label_layer_linear = nn.Sequential(nn.Linear(hidden_dim, hidden_dim), nn.Linear(hidden_dim, 19))
        self.color_layer_sine = FiLMLayer(hidden_dim + 3, hidden_dim)
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3))
        self.mapping_network = CustomMappingNetwork(z_dim, 256, (len(self.network) + 1) * hidden_dim * 2)

        for part in (self.network, self.final_layer, self.label_layer_linear, self.color_layer_sine,
                     self.color_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(first_layer_film_sine_init)
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        return FieldSpec(trunk_layers=len(self.network), color_layers=1, label_dim=19, grid_channels=0, grid_res=0,
                         input_scale=float(self.gridwarper.scale_factor), out_dim=23, double_latent=False)


class SPATIALSIRENSEMANTIC(TALLSIREN):
    """SPATIALSIRENBASELINE plus a label branch beside the colour branch (siren/siren.py:597-671): a FiLM layer on the
    trunk output, then Linear(256 -> 19).  FiLM rows: trunk 0..7, label 8, colour 9; output channels [labels (19),
    rgb (3), sigma (1)] whatever `output_dim` says."""

    def __init__(self, input_dim=2, z_dim=100, hidden_dim=256, output_dim=1, device=None):
        nn.Module.__init__(self)
        self.device = device
        self.input_dim = input_dim
        self.z_dim = z_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim
        self.max_batch_size = 2500

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        self.label_layer_sine = FiLMLayer(hidden_dim, hidden_dim)
        self.label_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 19))
        self.color_layer_sine = FiLMLayer(hidden_dim + 3, hidden_dim)
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3))
        self.mapping_network = CustomMappingNetwork(z_dim, 256, (len(self.network) + 2) * hidden_dim * 2)

        for part in (self.network, self.final_layer, self.label_layer_sine, self.label_layer_linear,
                     self.color_layer_sine, self.color_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(first_layer_film_sine_init)
        self.activation = nn.Softmax(dim=-1)     # unused, as in the reference (its forward returns raw logits)
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        return FieldSpec(trunk_layers=len(self.network), color_layers=1, label_dim=19, grid_channels=0, grid_res=0,
                         input_scale=float(self.gridwarper.scale_factor), out_dim=23, double_latent=False,
                         label_film=True)

    def film_rows(self):
        return len(self.network) + 2             # trunk, label, colour (siren.py:656-668)


class SPATIALSIRENBASELINEHD(TALLSIREN):
    """SPATIALSIRENBASELINE with a 64-feature colour head and no sigmoid (siren/siren.py:247-302), the field of a
    neural-renderer generator: output channels [features (64), sigma (1)] whatever `output_dim` says."""

    def __init__(self, input_dim=2, z_dim=100, hidden_dim=256, output_dim=1, device=None):
        nn.Module.__init__(self)
        self.device = device
        self.input_dim = input_dim
        self.z_dim = z_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        self.color_layer_sine = FiLMLayer(hidden_dim + 3, hidden_dim)
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 64))
        self.mapping_network = CustomMappingNetwork(z_dim, 256, (len(self.network) + 1) * hidden_dim * 2)

        for part in (self.network, self.final_layer, self.color_layer_sine, self.color_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(first_layer_film_sine_init)
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        return FieldSpec(trunk_layers=len(self.network), color_layers=1, label_dim=0, grid_channels=0, grid_res=0,
                         input_scale=float(self.gridwarper.scale_factor), out_dim=65, double_latent=False,
                         feature_head=True)


class SPATIALSIRENSEMANTICHD(SPATIALSIRENSEMANTIC):
    """SPATIALSIRENSEMANTIC with 64-wide heads (siren/siren.py:1301-1367): Linear(256 -> 64) label head and a 64-feature
    colour head without the sigmoid.  FiLM rows: trunk 0..7, label 8, colour 9; output channels [labels (64),
    features (64), sigma (1)] whatever `output_dim` says."""

    def __init__(self, input_dim=2, z_dim=100, hidden_dim=256, output_dim=1, device=None):
        nn.Module.__init__(self)
        self.device = device
        self.input_dim = input_dim
        self.z_dim = z_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim
        self.max_batch_size = 2500

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        self.label_layer_sine = FiLMLayer(hidden_dim, hidden_dim)
        self.label_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 64))
        self.color_layer_sine = FiLMLayer(hidden_dim + 3, hidden_dim)
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 64))
        self.mapping_network = CustomMappingNetwork(z_dim, 256, (len(self.network) + 2) * hidden_dim * 2)

        for part in (self.network, self.final_layer, self.label_layer_sine, self.label_layer_linear,
                     self.color_layer_sine, self.color_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(first_layer_film_sine_init)
        self.activation = nn.Softmax(dim=-1)     # unused, as in the reference
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        return FieldSpec(trunk_layers=len(self.network), color_layers=1, label_dim=64, grid_channels=0, grid_res=0,
                         input_scale=float(self.gridwarper.scale_factor), out_dim=129, double_latent=False,
                         label_film=True, feature_head=True)


class EmbeddingPiGAN256(TALLSIREN):
    """pi-GAN's embedding field at width 256 (siren/siren.py:341-410): a 32 x 64^3 feature grid feeds the first trunk
    layer, FiLM(cat[feat(32), pos(3)] -> 256), and not the colour branch, FiLM(cat[dir(3), x] -> 256).  FiLM rows: trunk
    0..7, colour 8; output channels [rgb (3), sigma (1)] whatever `output_dim` says.

    The reference builds it as EmbeddingPiGAN128.__init__(hidden_dim=256): that init draws a 32 x 96^3 grid (scaled by
    0.01) before this class replaces it with a 32 x 64^3 one (scaled by 0.1); both draws move the RNG, as here."""

    def __init__(self, input_dim=2, z_dim=100, hidden_dim=256, output_dim=1, device=None):
        nn.Module.__init__(self)
        self.device = device
        self.input_dim = input_dim
        self.z_dim = z_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim

        widths = [32 + 3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        print(self.network)
        self.final_layer = nn.Linear(hidden_dim, 1)
        self.color_layer_sine = FiLMLayer(hidden_dim + 3, hidden_dim)
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3))
        self.mapping_network = CustomMappingNetwork(z_dim, 256, (len(self.network) + 1) * hidden_dim * 2)

        for part in (self.network, self.final_layer, self.color_layer_sine, self.color_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(modified_first_sine_init)     # U(+-1/3) over all 35 columns
        torch.randn(1, 32, 96, 96, 96)                      # the 128-wide class's grid draw, replaced below
        self.gridwarper = UniformBoxWarp(0.24)
        self.spatial_embeddings = nn.Parameter(torch.randn(1, 32, 64, 64, 64) * 0.1)

    def field_spec(self):
        g = self.spatial_embeddings
        assert g.shape[2] == g.shape[3] == g.shape[4], "cubic feature grid expected"
        return FieldSpec(trunk_layers=len(self.network), color_layers=1, label_dim=0, grid_channels=g.shape[1],
                         grid_res=g.shape[2], input_scale=float(self.gridwarper.scale_factor), out_dim=4,
                         double_latent=False, grid_trunk=True)


class _DoubleLatentField(_FieldBase):
    """forward / FiLM-table plumbing shared by the double-latent (geometry, appearance) fields."""

    def film_table(self, frequencies_geo, frequencies_app, phase_shifts_geo, phase_shifts_app):
        """-> (B, L_geo + L_app, 2, 256) [15 f + 30, phase], geometry layers first (siren.py:1510-1511)."""
        b = frequencies_geo.shape[0]
        h = self.hidden_dim
        f = torch.cat([(frequencies_geo * 15 + 30).reshape(b, -1, h), (frequencies_app * 15 + 30).reshape(b, -1, h)], 1)
        p = torch.cat([phase_shifts_geo.reshape(b, -1, h), phase_shifts_app.reshape(b, -1, h)], 1)
        return torch.stack([f, p], dim=2).float().contiguous()

    def film_from_latents(self, z_geo, z_app, psi=1.0, avg=None):
        """(z_geo, z_app) -> FiLM table (geometry layers first); see TALLSIREN.film_from_latents.
        `avg` = (avg_frequencies_geo, avg_phase_shifts_geo, avg_frequencies_app, avg_phase_shifts_app)."""
        from .. import ops
        n_geo, n_app = len(self.network), len(self.color_layer_sine)
        if _fused_mapping_ok(self.geo_mapping_network, z_geo) and _fused_mapping_ok(self.app_mapping_network, z_app):
            film = torch.empty((z_geo.shape[0], n_geo + n_app, 2, self.hidden_dim), dtype=torch.float32, device=z_geo.device)
            ops.mapping_film(self.geo_mapping_network, z_geo, film, 0, n_geo, avg=None if avg is None else avg[0:2], psi=psi)
            return ops.mapping_film(self.app_mapping_network, z_app, film, n_geo, n_app, avg=None if avg is None else avg[2:4], psi=psi)
        f_geo, p_geo = self.geo_mapping_network(z_geo)
        f_app, p_app = self.app_mapping_network(z_app)
        if avg is not None:
            f_geo, p_geo = avg[0] + psi * (f_geo - avg[0]), avg[1] + psi * (p_geo - avg[1])
            f_app, p_app = avg[2] + psi * (f_app - avg[2]), avg[3] + psi * (p_app - avg[3])
        return self.film_table(f_geo, f_app, p_geo, p_app)

    def forward(self, input, z_geo, z_app, ray_directions, **kwargs):
        frequencies_geo, phase_shifts_geo = self.geo_mapping_network(z_geo)
        frequencies_app, phase_shifts_app = self.app_mapping_network(z_app)
        return self.forward_with_frequencies_phase_shifts(
            input, frequencies_geo, frequencies_app, phase_shifts_geo, phase_shifts_app, ray_directions, **kwargs)

    def forward_with_frequencies_phase_shifts(self, input, frequencies_geo, frequencies_app, phase_shifts_geo,
                                              phase_shifts_app, ray_directions, **kwargs):
        film = self.film_table(frequencies_geo, frequencies_app, phase_shifts_geo, phase_shifts_app)
        return self._render_points(input, film, ray_directions)


class SIRENBASELINESEMANTICDISENTANGLE(_DoubleLatentField):
    """TALLSIREN-style trunk with two latent codes and semantic logits, no feature grid
    (siren/siren.py:1163-1229); the network of the `CelebA_double_semantic` curriculum (curriculums.py:111).
    Output channels: [labels (output_dim-4), rgb (3), sigma (1)]; the label head is a two-Linear chain."""

    def __init__(self, input_dim=2, z_geo_dim=100, z_app_dim=100, hidden_dim=256, output_dim=1, device=None):
        super().__init__()
        self.device = device
        self.input_dim = input_dim
        self.z_geo_dim = z_geo_dim
        self.z_app_dim = z_app_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        cwidths = [hidden_dim + 3] + [hidden_dim] * 3
        self.color_layer_sine = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(cwidths[:-1], cwidths[1:]))
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3))
        self.geo_mapping_network = CustomMappingNetwork(z_geo_dim, 256, len(self.network) * hidden_dim * 2)
        self.app_mapping_network = CustomMappingNetwork(z_app_dim, 256, len(self.color_layer_sine) * hidden_dim * 2)
        self.label_layer_linear = nn.Sequential(nn.Linear(hidden_dim, hidden_dim), nn.Linear(hidden_dim, self.output_dim - 4))

        for part in (self.network, self.final_layer, self.color_layer_sine, self.color_layer_linear,
                     self.label_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(first_layer_film_sine_init)
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        return FieldSpec(trunk_layers=len(self.network), color_layers=len(self.color_layer_sine),
                         label_dim=self.output_dim - 4, grid_channels=0, grid_res=0,
                         input_scale=float(self.gridwarper.scale_factor), out_dim=self.output_dim, double_latent=True)


class SPATIALSIRENDISENTANGLE(_DoubleLatentField):
    """Geometry / appearance latents without a semantic head (siren/siren.py:747-813): 8 trunk FiLM layers on the
    geometry code, 3 colour FiLM layers on the appearance code, output [rgb, sigma]."""

    def __init__(self, input_dim=2, z_geo_dim=100, z_app_dim=100, hidden_dim=256, output_dim=1, device=None):
        super().__init__()
        self.device = device
        self.input_dim = input_dim
        self.z_geo_dim = z_geo_dim
        self.z_app_dim = z_app_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        cwidths = [hidden_dim + 3] + [hidden_dim] * 3
        self.color_layer_sine = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(cwidths[:-1], cwidths[1:]))
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3))
        self.geo_mapping_network = CustomMappingNetwork(z_geo_dim, 256, len(self.network) * hidden_dim * 2)
        self.app_mapping_network = CustomMappingNetwork(z_app_dim, 256, len(self.color_layer_sine) * hidden_dim * 2)

        for part in (self.network, self.final_layer, self.color_layer_sine, self.color_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(first_layer_film_sine_init)
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        return FieldSpec(trunk_layers=len(self.network), color_layers=len(self.color_layer_sine), label_dim=0,
                         grid_channels=0, grid_res=0, input_scale=float(self.gridwarper.scale_factor), out_dim=4,
                         double_latent=True)


class SPATIALSIRENSEMANTICDISENTANGLE(_DoubleLatentField):
    """The deep-appearance variant (siren/siren.py:1085-1161): 8 trunk + EIGHT colour FiLM layers, a two-Linear
    semantic head; the first colour layer gets the U(+-1/fan_in) first-layer init as well (:1131)."""

    def __init__(self, input_dim=2, z_geo_dim=100, z_app_dim=100, hidden_dim=256, output_dim=1, device=None):
        super().__init__()
        self.device = device
        self.input_dim = input_dim
        self.z_geo_dim = z_geo_dim
        self.z_app_dim = z_app_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        cwidths = [hidden_dim + 3] + [hidden_dim] * 8
        self.color_layer_sine = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(cwidths[:-1], cwidths[1:]))
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3))
        self.geo_mapping_network = CustomMappingNetwork(z_geo_dim, 256, len(self.network) * hidden_dim * 2)
        self.app_mapping_network = CustomMappingNetwork(z_app_dim, 256, len(self.color_layer_sine) * hidden_dim * 2)
        self.label_layer_linear = nn.Sequential(nn.Linear(hidden_dim, hidden_dim), nn.Linear(hidden_dim, self.output_dim - 4))

        for part in (self.network, self.final_layer, self.color_layer_sine, self.color_layer_linear,
                     self.label_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(first_layer_film_sine_init)
        self.color_layer_sine[0].apply(first_layer_film_sine_init)
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        return FieldSpec(trunk_layers=len(self.network), color_layers=len(self.color_layer_sine),
                         label_dim=self.output_dim - 4, grid_channels=0, grid_res=0,
                         input_scale=float(self.gridwarper.scale_factor), out_dim=self.output_dim, double_latent=True)


class TextureEmbeddingPiGAN128SEMANTICDISENTANGLE(_DoubleLatentField):
    """Double-latent field: geometry trunk + semantic head, texture branch with a 3-D feature grid
    (model B).  Output channels: [labels (output_dim-4), rgb (3), sigma (1)]."""

    def __init__(self, input_dim=2, z_geo_dim=100, z_app_dim=100, hidden_dim=128, output_dim=1, device=None):
        super().__init__()
        self.device = device
        self.input_dim = input_dim
        self.z_geo_dim = z_geo_dim
        self.z_app_dim = z_app_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        cwidths = [hidden_dim + 32 + 3] + [hidden_dim] * 3
        self.color_layer_sine = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(cwidths[:-1], cwidths[1:]))
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3))
        self.geo_mapping_network = CustomMappingNetwork(z_geo_dim, 256, len(self.network) * hidden_dim * 2)
        self.app_mapping_network = CustomMappingNetwork(z_app_dim, 256, len(self.color_layer_sine) * hidden_dim * 2)
        self.label_layer_linear = nn.Sequential(
            nn.Linear(hidden_dim, hidden_dim), nn.Linear(hidden_dim, hidden_dim),
            nn.Linear(hidden_dim, self.output_dim - 4))

        for part in (self.network, self.final_layer, self.color_layer_sine, self.color_layer_linear,
                     self.label_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(modified_first_sine_init)

        self.spatial_embeddings = nn.Parameter(torch.randn(1, 32, 96, 96, 96) * 0.01)
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        g = self.spatial_embeddings
        assert g.shape[2] == g.shape[3] == g.shape[4], "cubic feature grid expected"
        return FieldSpec(trunk_layers=len(self.network), color_layers=len(self.color_layer_sine),
                         label_dim=self.output_dim - 4, grid_channels=g.shape[1], grid_res=g.shape[2],
                         input_scale=float(self.gridwarper.scale_factor), out_dim=self.output_dim,
                         double_latent=True)


class TextureEmbeddingPiGAN256SEMANTICDISENTANGLE(TextureEmbeddingPiGAN128SEMANTICDISENTANGLE):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs, hidden_dim=256)
        self.spatial_embeddings = nn.Parameter(torch.randn(1, 32, 64, 64, 64) * 0.1)


class TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_DIM_96(TextureEmbeddingPiGAN128SEMANTICDISENTANGLE):
    """The production network of CelebA_double_semantic_texture_embedding_256_dim_96
    (curriculums.py:159): hidden 256, 32 x 96^3 grid."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs, hidden_dim=256)
        self.spatial_embeddings = nn.Parameter(torch.randn(1, 32, 96, 96, 96) * 0.1)


class SPATIALSIRENAUGDISENTANGLE(_DoubleLatentField):
    """SPATIALSIRENDISENTANGLE with a bridge between trunk and colour branch (siren/siren.py:904-979): v =
    color_layer_pre(x) is 3 wide, and 8 colour FiLM layers start from FiLM(cat[dir, v], 6 -> 256).  FiLM rows: trunk
    0..7, colour 8..15; output [rgb, sigma].  color_layer_pre keeps nn.Linear's default init, as in the reference."""

    def __init__(self, input_dim=2, z_geo_dim=100, z_app_dim=100, hidden_dim=256, output_dim=1, device=None):
        super().__init__()
        self.device = device
        self.input_dim = input_dim
        self.z_geo_dim = z_geo_dim
        self.z_app_dim = z_app_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim
        self.max_batch_size = 2500

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        self.color_layer_pre = nn.Sequential(nn.Linear(hidden_dim, 3))
        cwidths = [3 + 3] + [hidden_dim] * 8
        self.color_layer_sine = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(cwidths[:-1], cwidths[1:]))
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3))
        self.geo_mapping_network = CustomMappingNetwork(z_geo_dim, 256, len(self.network) * hidden_dim * 2)
        self.app_mapping_network = CustomMappingNetwork(z_app_dim, 256, len(self.color_layer_sine) * hidden_dim * 2)

        for part in (self.network, self.final_layer, self.color_layer_sine, self.color_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(first_layer_film_sine_init)
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        return FieldSpec(trunk_layers=len(self.network), color_layers=len(self.color_layer_sine), label_dim=0,
                         grid_channels=0, grid_res=0, input_scale=float(self.gridwarper.scale_factor), out_dim=4,
                         double_latent=True, bridge=True)


class RESSIRENDISENTANGLE(_DoubleLatentField):
    """The residual variant (siren/siren.py:982-1082): v = warped position + res_coord_layer(x); the density is
    density_layer_linear(v), four Linears without an activation, and 6 colour FiLM layers start from
    FiLM(cat[dir, color_layer_pre(v)], 259 -> 256).  No final_layer.  FiLM rows: trunk 0..7, colour 8..13; output
    [rgb, sigma].  res_coord_layer and color_layer_pre keep nn.Linear's default init, and the unused Softmax is kept, as
    in the reference."""

    def __init__(self, input_dim=2, z_geo_dim=100, z_app_dim=100, hidden_dim=256, output_dim=1, device=None):
        super().__init__()
        self.device = device
        self.input_dim = input_dim
        self.z_geo_dim = z_geo_dim
        self.z_app_dim = z_app_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim
        self.max_batch_size = 2500

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.res_coord_layer = nn.Linear(hidden_dim, 3)
        self.density_layer_linear = nn.Sequential(
            nn.Linear(3, hidden_dim), nn.Linear(hidden_dim, hidden_dim), nn.Linear(hidden_dim, hidden_dim),
            nn.Linear(hidden_dim, 1))
        self.color_layer_pre = nn.Sequential(nn.Linear(3, hidden_dim))
        cwidths = [hidden_dim + 3] + [hidden_dim] * 6
        self.color_layer_sine = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(cwidths[:-1], cwidths[1:]))
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3))
        self.geo_mapping_network = CustomMappingNetwork(z_geo_dim, 256, len(self.network) * hidden_dim * 2)
        self.app_mapping_network = CustomMappingNetwork(z_app_dim, 256, len(self.color_layer_sine) * hidden_dim * 2)

        for part in (self.network, self.density_layer_linear, self.color_layer_sine, self.color_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(first_layer_film_sine_init)
        self.activation = nn.Softmax(dim=-1)     # unused, as in the reference
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        return FieldSpec(trunk_layers=len(self.network), color_layers=len(self.color_layer_sine), label_dim=0,
                         grid_channels=0, grid_res=0, input_scale=float(self.gridwarper.scale_factor), out_dim=4,
                         double_latent=True, bridge=True, bridge_res=True)


class TextureEmbeddingPiGAN128SEMANTICDISENTANGLE_WO_DIR(_DoubleLatentField):
    """The direction-free sibling of model B (siren/siren.py:1549-1640): the same trunk, 32 x 96^3 grid and label chain,
    but EIGHT colour FiLM layers, the first on cat[feat(32), x] with no ray direction and the U(+-1/3)
    ``modified_first_sine_init`` (:1606).  FiLM rows: trunk 0..7, colour 8..15; output [labels, rgb, sigma].  The 128-wide
    class is here for name resolution, init and pickling: the kernels take hidden_dim=256 only."""

    def __init__(self, input_dim=2, z_geo_dim=100, z_app_dim=100, hidden_dim=128, output_dim=1, device=None):
        super().__init__()
        self.device = device
        self.input_dim = input_dim
        self.z_geo_dim = z_geo_dim
        self.z_app_dim = z_app_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim

        widths = [3] + [hidden_dim] * 8
        self.network = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(widths[:-1], widths[1:]))
        self.final_layer = nn.Linear(hidden_dim, 1)
        cwidths = [hidden_dim + 32] + [hidden_dim] * 8
        self.color_layer_sine = nn.ModuleList(FiLMLayer(a, b) for a, b in zip(cwidths[:-1], cwidths[1:]))
        self.color_layer_linear = nn.Sequential(nn.Linear(hidden_dim, 3))
        self.geo_mapping_network = CustomMappingNetwork(z_geo_dim, 256, len(self.network) * hidden_dim * 2)
        self.app_mapping_network = CustomMappingNetwork(z_app_dim, 256, len(self.color_layer_sine) * hidden_dim * 2)
        self.label_layer_linear = nn.Sequential(
            nn.Linear(hidden_dim, hidden_dim), nn.Linear(hidden_dim, hidden_dim),
            nn.Linear(hidden_dim, self.output_dim - 4))

        for part in (self.network, self.final_layer, self.color_layer_sine, self.color_layer_linear,
                     self.label_layer_linear):
            part.apply(frequency_init(25))
        self.network[0].apply(modified_first_sine_init)
        self.color_layer_sine[0].apply(modified_first_sine_init)     # U(+-1/3) over all 32 + hidden_dim columns

        self.spatial_embeddings = nn.Parameter(torch.randn(1, 32, 96, 96, 96) * 0.01)
        self.gridwarper = UniformBoxWarp(0.24)

    def field_spec(self):
        g = self.spatial_embeddings
        assert g.shape[2] == g.shape[3] == g.shape[4], "cubic feature grid expected"
        return FieldSpec(trunk_layers=len(self.network), color_layers=len(self.color_layer_sine),
                         label_dim=self.output_dim - 4, grid_channels=g.shape[1], grid_res=g.shape[2],
                         input_scale=float(self.gridwarper.scale_factor), out_dim=self.output_dim,
                         double_latent=True, wo_dir=True)


class TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96(TextureEmbeddingPiGAN128SEMANTICDISENTANGLE_WO_DIR):
    """The 256-wide production form (siren/siren.py:1817-1822): hidden 256, its own 32 x 96^3 grid (scaled by 0.1) drawn
    after the base class's (scaled by 0.01)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs, hidden_dim=256)
        self.spatial_embeddings = nn.Parameter(torch.randn(1, 32, 96, 96, 96) * 0.1)
