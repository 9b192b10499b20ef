"""Network containers with the interface of ``torchani.nn`` (nn/_core.py, nn/_containers.py).

``AtomicNetwork`` / ``ANINetworks`` / ``Ensemble`` hold ``torch.nn.Linear`` parameters with the
reference's module tree (so reference state dicts load: ``members.N.atomics.SYM.layers.K.weight``
/ ``final_layer``), while ``forward(elem_idxs, aevs, atomic, ensemble_values)`` runs the CUDA
grouped-GEMM kernels (``ani_b200_mlp_forward_backward``) on a species-grouped copy of the AEVs
and returns a tensor with an autograd edge to ``aevs`` (backward-to-input is produced by the
same kernel launch sequence; weights are inference-only, as in ``to_infer_model``).
"""
from __future__ import annotations

import ctypes as C
import typing as tp
import warnings

import torch
from torch import Tensor

from . import _lib
from ._lib import Grid, check, ptr
from .engine import PackedNetworks, TILE, operand_buffer, tile_a_operand

PERIODIC_TABLE = ("Dummy H He Li Be B C N O F Ne Na Mg Al Si P S Cl Ar K Ca Sc Ti V Cr Mn Fe Co Ni Cu Zn Ga "
                  "Ge As Se Br Kr Rb Sr Y Zr Nb Mo Tc Ru Rh Pd Ag Cd In Sn Sb Te I Xe").split()
ATOMIC_NUMBER = {s: i for i, s in enumerate(PERIODIC_TABLE)}


class SpeciesEnergies(tp.NamedTuple):
    species: Tensor
    energies: Tensor


class TightCELU(torch.nn.Module):
    r"""CELU activation function with alpha=0.1 (nn/_core.py:163-167)"""

    def forward(self, x: Tensor) -> Tensor:
        return torch.nn.functional.celu(x, alpha=0.1)


def activation_kind(activation: tp.Union[str, torch.nn.Module]) -> int:
    """The kernels' code of an activation: ``_lib.ACT_CELU`` for "celu" / a ``TightCELU`` (this package's or the
    reference's), ``_lib.ACT_GELU`` for "gelu" / ``torch.nn.GELU(approximate="none")``; ValueError otherwise."""
    if isinstance(activation, str):
        kinds = {"celu": _lib.ACT_CELU, "gelu": _lib.ACT_GELU}
        if activation not in kinds:
            raise ValueError(f"activation {activation!r}: the MLP kernels implement 'celu' (CELU(alpha=0.1)) and "
                             "'gelu' (exact-erf GELU) only")
        return kinds[activation]
    if type(activation).__name__ == "TightCELU":
        return _lib.ACT_CELU
    if type(activation) is torch.nn.GELU:
        if activation.approximate != "none":
            raise ValueError(f"GELU(approximate={activation.approximate!r}): the MLP kernels implement the exact-erf "
                             "GELU (approximate='none') only")
        return _lib.ACT_GELU
    raise ValueError(f"activation {activation!r}: the MLP kernels implement TightCELU (CELU(alpha=0.1)) and "
                     "torch.nn.GELU(approximate='none') only")


class AtomicNetwork(torch.nn.Module):
    """Parameter holder with the module tree of nn/_core.py:117-160.  The CUDA kernels support
    3 hidden layers + scalar output, in two kinds: CELU(0.1) with biases (the ANI-1x/2x/1ccx nets) and exact-erf
    GELU without biases (ANI-2xr / ANI-2dr and the models ``simple_ani`` assembles)."""

    def __init__(self, layer_dims: tp.Sequence[int], activation: tp.Union[str, torch.nn.Module] = "celu",
                 bias: bool = True) -> None:
        super().__init__()
        if any(d <= 0 for d in layer_dims):
            raise ValueError("Layer dims must be strict positive integers")
        kind = activation_kind(activation)
        if kind == _lib.ACT_CELU and not bias:
            raise ValueError("CELU networks without biases are not supported: the MLP kernels run CELU networks "
                             "with biases and GELU networks without")
        if kind == _lib.ACT_GELU and bias:
            raise ValueError("GELU networks with biases are not supported: the MLP kernels run GELU networks "
                             "without biases (bias=False) and CELU networks with")
        dims = tuple(layer_dims)
        self.layers = torch.nn.ModuleList(
            [torch.nn.Linear(i, o, bias=bias) for i, o in zip(dims[:-2], dims[1:-1])])
        self.final_layer = torch.nn.Linear(dims[-2], dims[-1], bias=bias)
        self.activation = TightCELU() if kind == _lib.ACT_CELU else torch.nn.GELU()
        self.has_biases = bias
        self.activation_kind = kind

    def linear_pairs(self) -> tp.List[tp.Tuple[Tensor, tp.Optional[Tensor]]]:
        return [(l.weight, l.bias) for l in list(self.layers) + [self.final_layer]]

    def forward(self, features: Tensor) -> Tensor:
        raise NotImplementedError("single AtomicNetworks are evaluated through their ANINetworks / Ensemble "
                                  "container on the CUDA path")


class _MLPFunction(torch.autograd.Function):
    """aevs (C, A, D) -> per-member atomic energies (M, C, A).  The backward-to-input for the
    ensemble mean is computed in the same pass and scaled by the upstream gradient."""

    @staticmethod
    def forward(ctx, aevs: Tensor, elem_idxs: Tensor, nets: PackedNetworks, want_grad: bool):
        dev = aevs.device
        n_conf, n_per_conf = elem_idxs.shape
        n = n_conf * n_per_conf
        S, M, D, ldx = nets.num_species, nets.num_members, nets.in_dim, nets.ldx
        flat = elem_idxs.reshape(-1)
        # order: real atoms first (stable), exactly what the layout kernel expects of a
        # bucket-sorted array; the "positions" here only carry the species
        order = torch.argsort((flat < 0).to(torch.int8), stable=True)
        sp_sorted = flat[order].to(torch.int32)
        spos = torch.zeros(n, 4, dtype=torch.float32, device=dev)
        spos[:, 3] = sp_sorted.view(torch.float32)
        grid = torch.zeros(C.sizeof(Grid) // 4, dtype=torch.int32, device=dev)
        grid[Grid.n_real.offset // 4] = (flat >= 0).sum().to(torch.int32)
        rows_cap = (n + S * (TILE - 1) + TILE - 1) // TILE * TILE
        i32 = dict(dtype=torch.int32, device=dev)
        row_of = torch.zeros(n, **i32)
        row_atom = torch.zeros(rows_cap, **i32)
        tile_species = torch.zeros(rows_cap // TILE, **i32)
        layout_info = torch.zeros(16, **i32)
        scratch = torch.zeros((n // 256 + 3) * 8 + 64, **i32)
        st = torch.cuda.current_stream(dev).cuda_stream
        L = _lib.lib(nets.variant)
        check(L.ani_b200_species_layout(ptr(spos), ptr(grid), n, 0, n, S, rows_cap, ptr(row_of), ptr(row_atom),
                                        ptr(tile_species), ptr(layout_info), ptr(scratch), st), "species_layout")
        xp = torch.zeros(rows_cap, ldx, dtype=torch.float32, device=dev)
        real = (sp_sorted >= 0)
        rows = torch.where(real, row_of, torch.zeros_like(row_of)).long()
        src = aevs.detach().reshape(n, D).to(torch.float32).index_select(0, order)
        src = src * real.view(-1, 1)
        # padding atoms all map to row 0 with zero contribution -> index_add keeps row 0 intact
        RLc, cp = nets.radial_len, nets.col_pad       # internal column order of the layer-1 operands (engine.PackedNetworks)
        if cp:
            xp[:, :RLc].index_add_(0, rows, src[:, :RLc])
            xp[:, RLc + cp:D + cp].index_add_(0, rows, src[:, RLc:])
        else:
            xp[:, :D].index_add_(0, rows, src)
        x_tiled = tile_a_operand(xp, variant=nets.variant)                    # the GEMM consumes the tiled form
        x = torch.zeros(rows_cap, ldx, dtype=torch.float32, device=dev)   # dE/dAEV comes back as plain rows
        act1, act2, act3 = (operand_buffer(rows_cap, w, dev, nets.variant) for w in nets.act_cols)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        e_member = torch.zeros(M, rows_cap, dtype=torch.float32, device=dev)
        check(L.ani_b200_mlp_forward_backward(C.byref(nets.model), ptr(x_tiled), ptr(x), rows_cap,
                                              ptr(row_atom), ptr(layout_info), None, ptr(act1), ptr(act2), ptr(act3),
                                              ptr(e_member), int(want_grad), ptr(status), st),
              "mlp_forward_backward")
        if int(status.item()) & _lib.STATUS_OPERAND_RANGE:   # this module-level path synchronises anyway
            raise _lib.OperandRangeError("an AEV, activation or gradient left the range of the half-precision GEMM "
                                         "operand pieces (inf/NaN input, or |value| > 1023.5 / |gradient| > 65504 / 4096)")
        em_sorted = e_member[:, rows] * real.view(1, -1)          # (M, n) in `order` order
        out = torch.zeros(M, n, dtype=torch.float32, device=dev)
        out[:, order] = em_sorted
        if want_grad:
            gx = x[rows]
            if cp:
                gx = torch.cat([gx[:, :RLc], gx[:, RLc + cp:D + cp]], 1)
            g_sorted = gx[:, :D] * real.view(-1, 1)                # d(mean energy)/d(aev), sorted order
            g = torch.zeros(n, D, dtype=torch.float32, device=dev)
            g[order] = g_sorted
            ctx.save_for_backward(g)
        ctx.shape = (n_conf, n_per_conf, D)
        ctx.scale = [nets.model.member_scale[m] for m in range(M)]
        ctx.want_grad = want_grad
        return out.view(M, n_conf, n_per_conf)

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        _lib.forbid_create_graph("the CUDA atomic networks (_MLPFunction)")
        if not ctx.want_grad:
            raise RuntimeError("this evaluation was run without the backward-to-input pass")
        (g,) = ctx.saved_tensors
        n_conf, n_per_conf, D = ctx.shape
        # the stored gradient is that of sum_m scale_m * e_m; it is valid when the upstream
        # gradient has the form grad_out[m, c, a] = scale_m * w[c, a]  (mean over members)
        scale = torch.tensor(ctx.scale, dtype=grad_out.dtype, device=grad_out.device).view(-1, 1, 1)
        active = scale.flatten() > 0
        w = (grad_out[active] / scale[active]).mean(0)
        if not torch.allclose(grad_out, scale * w.unsqueeze(0), rtol=1e-5, atol=1e-12):
            raise NotImplementedError("per-member gradients (ensemble_values=True backward) are not "
                                      "implemented on the CUDA path")
        return (g.view(n_conf, n_per_conf, D) * w.unsqueeze(-1)), None, None, None


class AtomicContainer(torch.nn.Module):
    r"""Base class for ANI modules that contain Atomic Neural Networks (nn/_core.py:68-115)"""

    num_species: int
    total_members_num: int
    active_members_idxs: tp.List[int]

    def __init__(self, *args: tp.Any, **kwargs: tp.Any) -> None:
        super().__init__()
        self.total_members_num = 1
        self.active_members_idxs = [0]
        self.num_species = 0
        self.register_buffer("atomic_numbers", torch.tensor([0], dtype=torch.long), persistent=False)
        self._packed: tp.Optional[PackedNetworks] = None
        self._packed_key: tp.Any = None
        self._packed_params: tp.Optional[tp.List[Tensor]] = None
        self._variant = ""   # operand-format build of the library ("" = 2 x fp16 pieces, "bf16x3"), see use_variant

    @property
    def symbols(self) -> tp.Tuple[str, ...]:
        return tuple(PERIODIC_TABLE[int(z)] for z in self.atomic_numbers)

    def get_active_members_num(self) -> int:
        return len(self.active_members_idxs)

    def set_active_members(self, idxs: tp.List[int]) -> None:
        for idx in idxs:
            if not (0 <= idx < self.total_members_num):
                raise IndexError(f"Idx {idx} should be 0 <= idx < {self.total_members_num}")
        self.active_members_idxs = list(idxs)
        if self._packed is not None:
            self._packed.set_active_members(self.active_members_idxs)

    def to_infer_model(self, use_mnp: bool = False) -> "AtomicContainer":
        return self  # already the inference-optimised container

    # -- weights in kernel layout ----------------------------------------------------------
    def member_networks(self) -> tp.List["ANINetworks"]:
        raise NotImplementedError

    def use_variant(self, variant: str) -> None:
        """Run this container on another operand-format build of the library ('bf16x3': three bfloat16 pieces per
        value -- 6 instead of 4 bytes per operand element, no range limit)."""
        if variant not in _lib.VARIANTS:
            raise ValueError(f"unknown library variant {variant!r}")
        if not _lib.available(variant):
            raise ImportError(f"{_lib.variant_path(variant)} has not been built (python -m torchani_b200.build)")
        if variant != self._variant:
            self._variant = variant
            self._packed_key = None

    def invalidate_packed(self) -> None:
        """Forget the kernel-layout copy of the weights (needed only after replacing ``p.data`` wholesale;
        in-place edits are seen through the parameters' version counters)."""
        self._packed_key = None
        self._packed_params = None

    def _apply(self, fn, *args, **kwargs):  # .to() / .cuda() / .float() ...
        self._packed_key = None
        self._packed_params = None
        return super()._apply(fn, *args, **kwargs)

    def _load_from_state_dict(self, *args, **kwargs) -> None:
        self._packed_key = None
        self._packed_params = None
        super()._load_from_state_dict(*args, **kwargs)

    def packed(self, device: torch.device) -> PackedNetworks:
        """Kernel-layout copy of the weights, rebuilt when a parameter was edited in place (the
        ``_version`` counters: optimizer steps, ``p.copy_()``, ...), replaced or moved."""
        if self._packed_params is None:
            self._packed_params = [p for m in self.member_networks() for p in m.parameters()]
        params = self._packed_params
        rl = getattr(self, "_radial_len", 0)   # set by the model that owns the AEV computer (models.ANI.engine)
        key = (str(device), self._variant, rl, tuple(p._version for p in params), tuple(p.data_ptr() for p in params[:2]))
        if self._packed is None or self._packed_key != key:
            members = self.member_networks()
            params = self._packed_params = [p for m in members for p in m.parameters()]
            key = (str(device), self._variant, rl, tuple(p._version for p in params),
                   tuple(p.data_ptr() for p in params[:2]))
            weights = [[self._packing_pairs(m.atomics[s]) for s in m.atomics] for m in members]
            in_dim = members[0].in_dim
            self._packed = PackedNetworks(weights, in_dim, device, variant=self._variant,
                                          radial_len=getattr(self, "_radial_len", 0),
                                          activation=members[0].activation_kind)
            self._packed.set_active_members(self.active_members_idxs)
            self._packed_key = key
        return self._packed

    def _packing_pairs(self, net: AtomicNetwork) -> tp.List[tp.Tuple[Tensor, tp.Optional[Tensor]]]:
        """The (W, b) pairs of a network as the kernels get them (``ChargeNetworks`` keeps one output row)."""
        return net.linear_pairs()

    def _run(self, elem_idxs: Tensor, aevs: Tensor, atomic: bool, ensemble_values: bool) -> Tensor:
        assert elem_idxs.shape == aevs.shape[:-1]
        if aevs.device.type != "cuda":
            raise ValueError("torchani_b200 runs on CUDA tensors only (there is no CPU path)")
        try:
            e_m = _MLPFunction.apply(aevs, elem_idxs, self.packed(aevs.device), bool(aevs.requires_grad))  # (M, C, A)
        except _lib.OperandRangeError:
            if not fall_back_to_bf16x3(self):
                raise
            e_m = _MLPFunction.apply(aevs, elem_idxs, self.packed(aevs.device), bool(aevs.requires_grad))
        nets = self._packed
        if ensemble_values:
            out = e_m[self.active_members_idxs]
            return out if atomic else out.sum(-1)
        scale = torch.tensor([nets.model.member_scale[m] for m in range(nets.num_members)],
                             dtype=e_m.dtype, device=e_m.device).view(-1, 1, 1)
        out = (e_m * scale).sum(0)
        return out if atomic else out.sum(-1)


def fall_back_to_bf16x3(*containers: AtomicContainer) -> bool:
    """The response to ANI_STATUS_OPERAND_RANGE (a value left the range of the 2 x fp16 operand pieces): False when the
    first container already runs on the 3 x bfloat16 build or that build is missing (the caller re-raises); otherwise
    warn, move every container to the 3 x bfloat16 build -- same kernels, 6 instead of 4 bytes per operand element, no
    range limit -- and return True (the caller redoes its work)."""
    if containers[0]._variant == "bf16x3" or not _lib.available("bf16x3"):
        return False
    warnings.warn("torchani_b200: operand range of the 2 x fp16 GEMM format exceeded; switching to the 3 x bfloat16 "
                  "build of the library")
    for c in containers:
        c.use_variant("bf16x3")
    return True


class ANINetworks(AtomicContainer):
    r"""Element-specific networks -> molecular or atomic scalars (nn/_containers.py:319-421)."""

    def __init__(self, modules: tp.Dict[str, AtomicNetwork], alias: bool = False):
        super().__init__()
        if any(s not in ATOMIC_NUMBER for s in modules):
            raise ValueError("All modules should be mapped to valid chemical symbols")
        if not alias and len(set(id(m) for m in modules.values())) != len(modules):
            raise ValueError("Symbols map to same module. If intended use `alias=True`")
        self.atomics = torch.nn.ModuleDict(modules)
        self.num_species = len(self.atomics)
        self.register_buffer("atomic_numbers",
                             torch.tensor([ATOMIC_NUMBER[e] for e in modules], dtype=torch.long), persistent=False)
        first = next(iter(self.atomics.values()))
        self.out_dim: int = first.final_layer.out_features
        self.in_dim: int = first.layers[0].in_features
        if len({m.activation_kind for m in self.atomics.values()}) != 1:
            raise ValueError("all networks of a container must share one activation (the MLP kernels run one per "
                             "model)")
        self.activation_kind: int = first.activation_kind

    def __getitem__(self, idx: str) -> AtomicNetwork:
        return self.atomics[idx]

    def member_networks(self) -> tp.List["ANINetworks"]:
        return [self]

    def forward(self, elem_idxs: Tensor, aevs: tp.Optional[Tensor] = None, atomic: bool = False,
                ensemble_values: bool = False) -> Tensor:
        if isinstance(elem_idxs, tuple):  # legacy call form nn/_containers.py:396-405
            warnings.warn("`ani_model((species, aevs))` is the TorchANI 1 signature; use `ani_model(species, aevs)`")
            return SpeciesEnergies(elem_idxs[0], self(elem_idxs[0], elem_idxs[1]))
        assert aevs is not None
        return self._run(elem_idxs, aevs, atomic, ensemble_values)

    # -- constructors (nn/_containers.py:423-570) ------------------------------------------
    @classmethod
    def build(cls, symbols: tp.Sequence[str], in_dim: int, dims: tp.Dict[str, tp.Tuple[int, ...]],
              out_dim: int = 1, activation: tp.Union[str, torch.nn.Module] = "gelu", bias: bool = False,
              default_dims: tp.Tuple[int, ...] = ()):
        return cls({s: AtomicNetwork((in_dim,) + tuple(dims.get(s, default_dims)) + (out_dim,), activation, bias)
                    for s in symbols})

    @classmethod
    def like_2x(cls, symbols: tp.Sequence[str] = ("H", "C", "N", "O", "S", "F", "Cl"), in_dim: int = 1008,
                out_dim: int = 1, activation: tp.Union[str, torch.nn.Module] = "celu", bias: bool = True):
        dims = {"H": (256, 192, 160), "C": (224, 192, 160), "N": (192, 160, 128), "O": (192, 160, 128),
                "S": (160, 128, 96), "F": (160, 128, 96), "Cl": (160, 128, 96)}
        return cls.build(symbols, in_dim, dims, out_dim, activation, bias, default_dims=(160, 128, 96))

    @classmethod
    def like_dr(cls, symbols: tp.Sequence[str] = ("H", "C", "N", "O", "S", "F", "Cl"), in_dim: int = 1008,
                out_dim: int = 1, activation: tp.Union[str, torch.nn.Module] = "gelu", bias: bool = False):
        """The networks of ANI-2dr (nn/_containers.py:447-478): GELU, no biases by default."""
        dims = {"H": (256, 192, 160), "C": (256, 192, 160), "N": (192, 160, 128), "O": (192, 160, 128),
                "S": (160, 128, 96), "F": (160, 128, 96), "Cl": (160, 128, 96)}
        return cls.build(symbols, in_dim, dims, out_dim, activation, bias, default_dims=(160, 128, 96))

    @classmethod
    def default(cls, symbols: tp.Sequence[str], in_dim: int, out_dim: int = 1,
                activation: tp.Union[str, torch.nn.Module] = "gelu", bias: bool = False):
        """The networks ``simple_ani`` assembles (nn/_containers.py:531-540): ANI-2x widths, GELU, no biases."""
        return cls.like_2x(symbols, in_dim, out_dim, activation, bias)

    @classmethod
    def like_1x(cls, symbols: tp.Sequence[str] = ("H", "C", "N", "O"), in_dim: int = 384, out_dim: int = 1,
                activation: tp.Union[str, torch.nn.Module] = "celu", bias: bool = True):
        dims = {"H": (160, 128, 96), "C": (144, 112, 96), "N": (128, 112, 96), "O": (128, 112, 96)}
        return cls.build(symbols, in_dim, dims, out_dim, activation, bias, default_dims=(128, 112, 96))


class ChargeNetworks(ANINetworks):
    r"""Element-specific networks -> raw atomic charges, the charge networks of an ANIq model (potentials/nnp.py:75-102).

    Two forms of the reference share this container and its module tree (``atomics.SYM.layers.K.weight``,
    ``atomics.SYM.final_layer.weight``):

    * ``ANINetworks`` with ``out_dim = 1`` (``simple_aniq``, arch.py:1071-1182): ``kept_output = 0``;
    * ``_ANINetworksDiscardFirstScalar`` with ``out_dim = 2`` (ANImbis, nn/_internal.py:69-90): only output column 1
      is used, ``kept_output = 1``.

    The kernels get the kept row of every final layer.  Charges carry no gradient: ``forward`` evaluates the networks
    forward-only."""

    def __init__(self, modules: tp.Dict[str, AtomicNetwork], alias: bool = False, kept_output: tp.Optional[int] = None):
        super().__init__(modules, alias)
        if kept_output is None:
            kept_output = 1 if self.out_dim == 2 else 0
        if (self.out_dim, kept_output) not in ((1, 0), (2, 1)):
            raise ValueError("charge networks have out_dim = 1, or out_dim = 2 of which column 1 is the charge "
                             f"(_ANINetworksDiscardFirstScalar); got out_dim = {self.out_dim}, column {kept_output}")
        self.kept_output = int(kept_output)

    def _packing_pairs(self, net: AtomicNetwork) -> tp.List[tp.Tuple[Tensor, tp.Optional[Tensor]]]:
        pairs = net.linear_pairs()
        k = self.kept_output
        w, b = pairs[-1]
        return pairs[:-1] + [(w[k:k + 1], None if b is None else b[k:k + 1])]

    def forward(self, elem_idxs: Tensor, aevs: tp.Optional[Tensor] = None, atomic: bool = True,
                ensemble_values: bool = False) -> Tensor:
        """Raw charges (C, A), 0 for padding atoms (or their sums per conformer with ``atomic=False``)."""
        assert aevs is not None
        return self._run(elem_idxs, aevs.detach(), atomic, False)

    @classmethod
    def like_2x(cls, symbols: tp.Sequence[str] = ("H", "C", "N", "O", "S", "F", "Cl"), in_dim: int = 1008,
                out_dim: int = 2, activation: tp.Union[str, torch.nn.Module] = "gelu", bias: bool = False):
        """ANImbis's charge networks (models.py:201-252): ANI-2x widths, GELU, no biases, ``out_dim = 2``."""
        return super().like_2x(symbols, in_dim, out_dim, activation, bias)


class ANIModel(ANINetworks):
    """Deprecated alias kept by the reference (nn/_internal.py:13-19)."""

    def __init__(self, modules: tp.Any):
        if not isinstance(modules, dict):
            raise ValueError("torchani_b200.nn.ANIModel needs a {symbol: AtomicNetwork} mapping")
        super().__init__(modules, alias=True)


class Ensemble(AtomicContainer):
    r"""Average over many containers of networks (nn/_containers.py:573-660)."""

    def __init__(self, modules: tp.Iterable[ANINetworks], repeats: bool = False):
        super().__init__()
        modules = list(modules)
        if not repeats and len(set(map(id, modules))) != len(modules):
            raise ValueError("Modules are repeated. If intended use `repeats=True`")
        self.members = torch.nn.ModuleList(modules)
        self.total_members_num = len(self.members)
        self.active_members_idxs = list(range(self.total_members_num))
        self.num_species = modules[0].num_species
        if any(m.num_species != self.num_species for m in modules):
            raise ValueError("All modules must support the same number of elements")
        if any(m.activation_kind != modules[0].activation_kind for m in modules):
            raise ValueError("all members of an ensemble must share one activation (the MLP kernels run one per "
                             "model)")
        self.register_buffer("atomic_numbers", modules[0].atomic_numbers, persistent=False)

    def __len__(self) -> int:
        return self.total_members_num

    def __getitem__(self, idx: int) -> ANINetworks:
        return tp.cast(ANINetworks, self.members[idx])

    def member_networks(self) -> tp.List[ANINetworks]:
        return list(self.members)

    def forward(self, elem_idxs: Tensor, aevs: tp.Optional[Tensor] = None, atomic: bool = False,
                ensemble_values: bool = False) -> Tensor:
        if isinstance(elem_idxs, tuple):  # legacy call form nn/_containers.py:615-624
            warnings.warn("`ensemble((species, aevs))` is the TorchANI 1 signature; use `ensemble(species, aevs)`")
            return SpeciesEnergies(elem_idxs[0], self(elem_idxs[0], elem_idxs[1]))
        assert aevs is not None
        return self._run(elem_idxs, aevs, atomic, ensemble_values)


class SpeciesConverter(torch.nn.Module):
    r"""Convert atomic numbers into internal ANI element indices (nn/_containers.py:663-734)"""

    conv_tensor: Tensor

    def __init__(self, symbols: tp.Sequence[str]):
        super().__init__()
        if isinstance(symbols, str):
            raise ValueError("Please use 'SpeciesConverter(['H', 'C', 'N', 'O'])' instead")
        self.register_buffer("conv_tensor", torch.full((len(PERIODIC_TABLE) + 1,), -1, dtype=torch.long))
        for i, s in enumerate(symbols):
            self.conv_tensor[ATOMIC_NUMBER[s]] = i
        self.atomic_numbers = torch.tensor([ATOMIC_NUMBER[e] for e in symbols], dtype=torch.long)

    def forward(self, atomic_nums: Tensor, nop: bool = False) -> Tensor:
        if isinstance(atomic_nums, tuple):
            warnings.warn("`converter((atomic_nums, coords))` is the TorchANI 1 signature")
            return (self(atomic_nums[0]), atomic_nums[1])
        if nop:
            if atomic_nums.max() >= len(self.atomic_numbers):
                raise ValueError(f"Unsupported element idx in {atomic_nums}")
            return atomic_nums
        elem_idxs = self.conv_tensor[atomic_nums]
        if (elem_idxs[atomic_nums != -1] == -1).any():
            raise ValueError(
                f"Model doesn't support some elements in input Input elements include: "
                f"{torch.unique(atomic_nums)} Supported elements are: {self.atomic_numbers}")
        return elem_idxs
