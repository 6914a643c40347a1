"""Host glue between a field module (fenerf_b200.siren.siren) and ``fenerf_pack_field``.

Collects the raw ``nn.Parameter`` device pointers into ``fenerf_field_params`` and lets the library
re-lay them out on the device; PyTorch only owns the memory.
"""
import ctypes as C
from dataclasses import dataclass

import torch

from . import _lib


@dataclass
class PackedField:
    desc: "_lib.FieldDesc"
    buffer: torch.Tensor      # owning uint8 allocation
    ptr: int                  # 1024-byte aligned device pointer inside `buffer`
    nbytes: int
    device: torch.device
    stream: int = 0               # cuda stream the pack kernels ran on
    event: "torch.cuda.Event" = None   # recorded after them: consumers on another stream wait on it
    fingerprint: tuple = None     # (u64, u64) of the raw parameters at pack time, filled lazily

    def wait_ready(self):
        """Orders the caller's current stream after the pack kernels when it is a different stream."""
        if self.event is None or torch.cuda.is_current_stream_capturing():
            return      # (graph capture follows a warm-up + device synchronize, fenerf_b200/graphs.py: the pack is long done)
        cur = torch.cuda.current_stream(self.device)
        if cur.cuda_stream != self.stream:
            if self.event.query():           # long finished (the steady state; also keeps graph capture clean)
                self.event = None
            else:
                cur.wait_event(self.event)


def field_desc(spec, split=False) -> "_lib.FieldDesc":
    return _lib.FieldDesc(trunk_layers=spec.trunk_layers, color_layers=spec.color_layers, label_dim=spec.label_dim,
                          grid_channels=spec.grid_channels, grid_res=spec.grid_res, out_dim=spec.out_dim,
                          input_scale=spec.input_scale,
                          reserved=(_lib.FIELD_LABEL_FILM if spec.label_film else 0)
                          | (_lib.FIELD_FEATURE_HEAD if spec.feature_head else 0)
                          | (_lib.FIELD_GRID_TRUNK if spec.grid_trunk else 0)
                          | (_lib.FIELD_BRIDGE if spec.bridge else 0)
                          | (_lib.FIELD_BRIDGE_RES if spec.bridge_res else 0)
                          | (_lib.FIELD_WO_DIR if spec.wo_dir else 0)
                          | (_lib.FIELD_SPLIT_IMAGES if split else 0))


def _f32(t, device):
    t = t.detach()
    if t.dtype != torch.float32 or not t.is_contiguous() or t.device != device:
        t = t.to(device=device, dtype=torch.float32).contiguous()
    return t


def collect_params(module, device):
    """-> (FieldParams, BridgeParams or None, keepalive list). Parameter order / names per SURVEY.md section 8b."""
    spec = module.field_spec()
    if getattr(module, "hidden_dim", 256) != _lib.HIDDEN:
        raise ValueError("the sm_90a kernels are specialised for hidden_dim=256 (got %s)" % module.hidden_dim)
    keep = []

    def ptr(t):
        t = _f32(t, device)
        keep.append(t)
        return t.data_ptr()

    p = _lib.FieldParams()
    for i, layer in enumerate(module.network):
        p.trunk_w[i] = ptr(layer.layer.weight)
        p.trunk_b[i] = ptr(layer.layer.bias)
    if not spec.bridge_res:      # (RESSIRENDISENTANGLE has no final_layer: its density is a chain on v)
        p.sigma_w = ptr(module.final_layer.weight)
        p.sigma_b = ptr(module.final_layer.bias)
    color = module.color_layer_sine
    color = list(color) if isinstance(color, torch.nn.ModuleList) else [color]
    for i, layer in enumerate(color):
        p.color_w[i] = ptr(layer.layer.weight)
        p.color_b[i] = ptr(layer.layer.bias)
    p.rgb_w = ptr(module.color_layer_linear[0].weight)
    p.rgb_b = ptr(module.color_layer_linear[0].bias)
    if spec.label_film:
        # slots: [label FiLM layer, NULL, head 256->label_dim] (include/fenerf_b200.h, FENERF_FIELD_LABEL_FILM)
        head = [m for m in module.label_layer_linear if isinstance(m, torch.nn.Linear)]
        if len(head) != 1:
            raise ValueError("label FiLM head: expected one Linear layer, got %d" % len(head))
        for i, lin in ((0, module.label_layer_sine.layer), (2, head[0])):
            p.label_w[i] = ptr(lin.weight)
            p.label_b[i] = ptr(lin.bias)
    elif spec.label_dim:
        chain = [m for m in module.label_layer_linear if isinstance(m, torch.nn.Linear)]
        if len(chain) not in (2, 3):
            raise ValueError("label head: expected a chain of 2 or 3 Linear layers, got %d" % len(chain))
        # slots: [first 256->256, middle 256->256 or absent, last 256->label_dim]
        slots = {0: chain[0], 2: chain[-1]}
        if len(chain) == 3:
            slots[1] = chain[1]
        for i, lin in slots.items():
            p.label_w[i] = ptr(lin.weight)
            p.label_b[i] = ptr(lin.bias)
    if spec.grid_channels:
        p.grid = ptr(module.spatial_embeddings)
    bridge = None
    if spec.bridge:
        # v = Linear(256 -> 3) of the trunk output: color_layer_pre, or res_coord_layer with the density chain
        lin = module.res_coord_layer if spec.bridge_res else module.color_layer_pre[0]
        p.label_w[0] = ptr(lin.weight)
        p.label_b[0] = ptr(lin.bias)
    if spec.bridge_res:
        bridge = _lib.BridgeParams()
        for i, lin in enumerate(module.density_layer_linear):
            bridge.density_w[i] = ptr(lin.weight)
            bridge.density_b[i] = ptr(lin.bias)
        bridge.pre_w = ptr(module.color_layer_pre[0].weight)
        bridge.pre_b = ptr(module.color_layer_pre[0].bias)
    return p, bridge, keep


def _bridge_ref(bridge):
    return C.byref(bridge) if bridge is not None else None


def pack_field(module, split=False) -> PackedField:
    """split=True: the layout with the fp16 low parts of the weight images that precision='split' reads
    (FENERF_FIELD_SPLIT_IMAGES)."""
    lib = _lib.lib()
    device = next(module.parameters()).device
    if device.type != "cuda":
        raise RuntimeError("fenerf_b200 renders on CUDA only; move the generator to an H100 (got %s)" % device)
    spec = module.field_spec()
    desc = field_desc(spec, split)
    nbytes = lib.fenerf_packed_bytes(C.byref(desc))
    if nbytes == 0:
        _lib.check(-1)
    with torch.cuda.device(device):
        buf = torch.empty(nbytes + 1024, dtype=torch.uint8, device=device)
        ptr = (buf.data_ptr() + 1023) // 1024 * 1024
        params, bridge, keep = collect_params(module, device)
        stream = torch.cuda.current_stream(device).cuda_stream
        _lib.check(lib.fenerf_pack_field_bridge(C.byref(desc), C.byref(params), _bridge_ref(bridge), ptr, nbytes, stream))
        event = torch.cuda.Event()
        event.record()
        del keep
    return PackedField(desc=desc, buffer=buf, ptr=ptr, nbytes=nbytes, device=device, stream=stream, event=event)


def fingerprint(module):
    """(u64, u64) fingerprint of the field's raw parameters -- one kernel + a 16-byte read-back, i.e. a
    host synchronisation: used where the caller synchronises anyway (staged_forward*, whose outputs go to
    the CPU) to catch parameter writes that bypass torch's version counters (torch_ema ``copy_to`` /
    ``restore`` use ``param.data.copy_``)."""
    lib = _lib.lib()
    device = next(module.parameters()).device
    desc = field_desc(module.field_spec())
    with torch.cuda.device(device):
        out = torch.empty(2, dtype=torch.int64, device=device)
        params, bridge, keep = collect_params(module, device)
        _lib.check(lib.fenerf_field_fingerprint_bridge(C.byref(desc), C.byref(params), _bridge_ref(bridge), out.data_ptr(),
                                                       torch.cuda.current_stream(device).cuda_stream))
        a, b = out.tolist()
        del keep
    return a, b
