"""Host side of the fused hot path: owns the device workspaces (the C-ABI never allocates) and
sequences the kernels of ``libani_b200.so`` on the current CUDA stream.

One step  =  bucket grid -> species layout -> fused neighbour search + AEV -> ensemble MLP
forward + backward-to-AEV -> AEV backward (dE/dcoords) -> energy reduction.  No host
synchronisation happens inside a step; device-side error conditions accumulate in a status
word that is checked when results are read (``Engine.check_status``).

PyTorch is used only for device memory, streams and (in ``parallel.py``) torch.distributed.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import typing as tp

import numpy as np
import torch
from torch import Tensor

from . import _lib
from ._lib import AEVParams, D3Params, Grid, MLPModel, PairParams, check, ptr

TILE = _lib.ANI_TILE_ROWS


def _f32(v: float) -> float:
    return float(np.float32(v))


class AEVConstants(tp.NamedTuple):
    """The numbers that define an ANI AEV (see aev/_computer.py:499-600 in the reference)."""

    num_species: int
    rcr: float
    rca: float
    eta_r: float
    shf_r: tp.Tuple[float, ...]
    eta_a: float
    zeta: float
    shf_a: tp.Tuple[float, ...]
    shf_z: tp.Tuple[float, ...]
    cutoff_fn: str = "cosine"

    @property
    def radial_len(self) -> int:
        return self.num_species * len(self.shf_r)

    @property
    def angular_len(self) -> int:
        return self.num_species * (self.num_species + 1) // 2 * len(self.shf_a) * len(self.shf_z)

    @property
    def out_dim(self) -> int:
        return self.radial_len + self.angular_len

    def to_struct(self) -> AEVParams:
        if self.cutoff_fn not in ("cosine", "smooth"):
            raise ValueError(f"cutoff function {self.cutoff_fn!r} is not supported by the CUDA kernels")
        if (len(self.shf_a), len(self.shf_z)) not in ((8, 4), (4, 8)):
            raise ValueError("the AEV kernels need ShfA x ShfZ = 8x4 (ANI-2x) or 4x8 (ANI-1x)")
        if len(self.shf_r) > _lib.ANI_MAX_SHFR or self.num_species > _lib.ANI_MAX_SPECIES:
            raise ValueError("too many radial shifts / species for the CUDA kernels")
        p = AEVParams()
        p.rcr, p.rca = self.rcr, self.rca
        # the reference keeps eta/zeta/shifts as float32 buffers (aev/_terms.py:153-156,288-292)
        p.eta_r, p.eta_a, p.zeta = _f32(self.eta_r), _f32(self.eta_a), _f32(self.zeta)
        p.n_shf_r, p.n_shf_a, p.n_shf_z = len(self.shf_r), len(self.shf_a), len(self.shf_z)
        p.num_species = self.num_species
        p.cutoff_kind = 0 if self.cutoff_fn == "cosine" else 1
        for k, v in enumerate(self.shf_r):
            p.shf_r[k] = _f32(v)
        for k, v in enumerate(self.shf_a):
            p.shf_a[k] = _f32(v)
        for k, v in enumerate(self.shf_z):
            p.cos_z[k] = math.cos(_f32(v))
            p.sin_z[k] = math.sin(_f32(v))
        return p


def _linspace(start: float, stop: float, steps: int) -> tp.Tuple[float, ...]:
    return tuple(start + ((stop - start) / steps) * j for j in range(steps))  # utils.py:101-107


def constants_2x(num_species: int = 7, cutoff_fn: str = "cosine") -> AEVConstants:
    a0 = math.pi / 4 / 2
    return AEVConstants(num_species, 5.1, 3.5, 19.7, _linspace(0.8, 5.1, 16), 12.5, 14.1,
                        _linspace(0.8, 3.5, 8), _linspace(a0, math.pi + a0, 4), cutoff_fn)


def constants_1x(num_species: int = 4, cutoff_fn: str = "cosine") -> AEVConstants:
    a0 = math.pi / 8 / 2
    return AEVConstants(num_species, 5.2, 3.5, 16.0, _linspace(0.9, 5.2, 16), 8.0, 32.0,
                        _linspace(0.9, 3.5, 4), _linspace(a0, math.pi + a0, 8), cutoff_fn)


def _split(x: Tensor, scale: float = 1.0, variant: tp.Optional[str] = None) -> tp.List[Tensor]:
    """x (float32) -> the 16-bit pieces of ``scale * x`` in the library's operand format
    (``_lib.operand_format``): two IEEE half pieces or three bfloat16 pieces, each rounded to
    nearest, ``scale * x = p1 + p2 (+ p3)``."""
    fmt = _lib.operand_format(variant)
    dt = torch.float16 if fmt.parts == 2 else torch.bfloat16
    r = x.to(torch.float32) * scale
    out = []
    for _ in range(fmt.parts):
        p = r.to(dt)
        out.append(p)
        r = r - p.to(torch.float32)
    return out


def weight_scale(ws: tp.Sequence[Tensor], variant: tp.Optional[str] = None) -> float:
    """Power-of-two operand scale for a group of weight matrices (half pieces: the largest
    |scale * w| stays below 2^14, the scale below 2^12; bfloat16 pieces need none)."""
    if _lib.operand_format(variant).parts != 2:
        return 1.0
    top = max(float(w.abs().max()) for w in ws)
    if not math.isfinite(top):
        raise ValueError("network weights contain inf/NaN")
    if top == 0.0:
        return 4096.0
    return float(min(4096.0, max(1.0, 2.0 ** math.floor(math.log2(16384.0 / top)))))


def _swizzle_index(device) -> Tensor:
    """idx[row in 8-row group][position] = the 16-byte chunk stored at that position (SWIZZLE_64B)."""
    rows = torch.arange(8, device=device).view(8, 1)
    pos = torch.arange(4, device=device).view(1, 4)
    return pos ^ ((rows >> 1) & 3)


def tile_b_operand(b: Tensor, scale: float = 1.0, variant: tp.Optional[str] = None) -> Tensor:
    """``B[N][K]`` (float32, K-major, N % 32 == 0) -> the "tiled B operand" byte layout of
    include/ani_b200.h: K zero-padded to 32, the 16-bit pieces of ``scale * B``,
    [n tile of 256 rows][k block of 32][p1 bn x 64 B | p2 (| p3)] with every 8-row group in wgmma
    SWIZZLE_64B order.  Returned as a flat 16-bit tensor."""
    n, k = b.shape
    assert n % 32 == 0, "rows of a B operand must come in groups of 32"
    kp = (k + 31) // 32 * 32
    nkb = kp // 32
    bp = torch.zeros(n, kp, dtype=torch.float32, device=b.device)
    bp[:, :k] = b
    pieces = _split(bp, scale, variant)
    src_chunk = _swizzle_index(b.device)
    out = []
    for n0 in range(0, n, 256):
        bn = min(256, n - n0)
        parts = []
        idx = src_chunk.view(1, 1, 8, 4, 1).expand(nkb, bn // 8, 8, 4, 8)
        for part in pieces:
            x = part[n0:n0 + bn].view(bn // 8, 8, nkb, 4, 8)           # [group][row][kb][chunk][8]
            x = x.permute(2, 0, 1, 3, 4)                                # [kb][group][row][chunk][8]
            parts.append(torch.gather(x, 3, idx).reshape(nkb, bn * 32))
        out.append(torch.stack(parts, 1).reshape(-1))                  # [kb][piece][bn*32]
    return torch.cat(out).contiguous()


def tile_a_operand(x: Tensor, scale: tp.Optional[float] = None, variant: tp.Optional[str] = None) -> Tensor:
    """Plain ``[rows][cols]`` float32 (rows % 128 == 0, cols % 32 == 0) -> flat "tiled operand"
    (A-operand form of include/ani_b200.h; ``scale`` defaults to the library's value scale).
    Plumbing for the API paths that receive plain AEVs."""
    rows, cols = x.shape
    assert rows % 128 == 0 and cols % 32 == 0
    nkb = cols // 32
    if scale is None:
        scale = _lib.operand_format(variant).value_scale
    idx = _swizzle_index(x.device).view(1, 1, 1, 8, 4, 1).expand(rows // 128, nkb, 16, 8, 4, 8)
    parts = []
    for part in _split(x.contiguous().to(torch.float32), scale, variant):
        v = part.view(rows // 128, 16, 8, nkb, 4, 8).permute(0, 3, 1, 2, 4, 5)   # [rt][kb][grp][row][ch][8]
        parts.append(torch.gather(v, 4, idx).reshape(rows // 128, nkb, 4096))
    return torch.stack(parts, 2).reshape(-1).contiguous()                          # [rt][kb][piece][4096]


def untile_a_operand(t: Tensor, rows: int, cols: int, scale: tp.Optional[float] = None,
                     variant: tp.Optional[str] = None) -> Tensor:
    """Inverse of ``tile_a_operand`` (returns (p1 + p2 (+ p3)) / scale as plain float32 ``[rows][cols]``)."""
    fmt = _lib.operand_format(variant)
    if scale is None:
        scale = fmt.value_scale
    nkb = cols // 32
    P = fmt.parts
    dt = torch.float16 if P == 2 else torch.bfloat16
    v = t.view(dt).view(rows // 128, nkb, P, 16, 8, 4, 8)                        # [rt][kb][piece][grp][row][pos][8]
    idx = _swizzle_index(t.device).view(1, 1, 1, 1, 8, 4, 1).expand(rows // 128, nkb, P, 16, 8, 4, 8)
    w = torch.gather(v.to(torch.float32), 5, idx).flip(2).sum(2) / scale           # [rt][kb][grp][row][ch][8]
    return w.permute(0, 2, 3, 1, 4, 5).reshape(rows, cols).contiguous()


def operand_buffer(rows: int, cols: int, device, variant: tp.Optional[str] = None) -> Tensor:
    """Zeroed storage of a tiled operand matrix with ``rows x cols`` values."""
    fmt = _lib.operand_format(variant)
    return torch.zeros(rows, fmt.parts * cols, dtype=torch.float16 if fmt.parts == 2 else torch.bfloat16,
                       device=device)


class PackedNetworks:
    """Device-resident, kernel-layout copy of an ensemble of per-element MLPs (``dims`` keeps the
    true layer widths, the kernel model the widths padded to multiples of 32).

    ``weights[member][species_index] = [(W [out,in], b [out]) x 4]`` in ``torch.nn.Linear``
    layout (nn/_core.py:117-149).  All members must share the layer widths of a species.
    ``activation``: ``_lib.ACT_CELU`` (CELU(celu_alpha), every ``b`` given) or ``_lib.ACT_GELU`` (GELU, every ``b``
    None: bias-free networks, the kernel model gets zeros it never reads).
    """

    def __init__(self, weights: tp.Sequence[tp.Sequence[tp.Sequence[tp.Tuple[Tensor, tp.Optional[Tensor]]]]],
                 in_dim: int, device: torch.device, celu_alpha: float = 0.1, variant: tp.Optional[str] = None,
                 radial_len: int = 0, activation: int = _lib.ACT_CELU):
        """``radial_len`` (number of radial AEV columns, S * len(ShfR)) > 0 and not a multiple of 32: the angular block
        of the layer-1 operands starts at the next 32-column boundary (``col_pad`` zero columns in between) if that
        still fits the padded width -- every element pair then fills exactly one 32-column GEMM block, and the
        block-sparse layer 1 skips more (water: 5 live blocks instead of 8).  The AEV kernels write / read the same
        internal order (``ani_aev_params::ang_pad``); plain AEV rows keep the reference's order."""
        self.device = torch.device(device)
        self.variant = variant or ""   # build of the library (operand format) these operands are packed for
        M = len(weights)
        S = len(weights[0])
        if not (1 <= M <= _lib.ANI_MAX_MEMBERS) or not (1 <= S <= _lib.ANI_MAX_SPECIES):
            raise ValueError("unsupported number of ensemble members / species")
        self.num_members, self.num_species, self.in_dim = M, S, in_dim
        self.ldx = (in_dim + 31) // 32 * 32
        self.radial_len = int(radial_len)
        self.col_pad = (-self.radial_len) % 32 if 0 < self.radial_len < in_dim else 0
        if in_dim + self.col_pad > self.ldx or os.environ.get("ANI_B200_ALIGN_ANGULAR", "1") == "0":
            self.col_pad = 0
        self.celu_alpha = celu_alpha
        if activation not in (_lib.ACT_CELU, _lib.ACT_GELU):
            raise ValueError(f"unknown activation {activation!r} (engine: _lib.ACT_CELU or _lib.ACT_GELU)")
        self.activation = activation
        self.dims: tp.List[tp.Tuple[int, int, int]] = []
        self._keep: tp.List[Tensor] = []
        self.model = MLPModel()
        mdl = self.model
        mdl.num_species, mdl.num_members, mdl.in_dim, mdl.ldx = S, M, in_dim, self.ldx
        mdl.celu_alpha = celu_alpha
        mdl.activation = activation
        # Weights are gathered on the HOST into one flat float32 buffer (zero-padded to 32-column blocks),
        # uploaded with a single copy and re-laid out into the tiled B operands by this library's own
        # ani_b200_pack_b_operand kernel: no ATen kernel touches them (one launch per operand kind).
        pad = lambda v: (v + 31) // 32 * 32  # noqa: E731
        P2 = 2 * _lib.operand_format(self.variant).parts          # bytes per operand element
        plan = []                                     # per species: sizes, scales, source / destination offsets
        src_off = 0
        dst_off = 0

        def take_src(count: int) -> int:
            nonlocal src_off
            o = src_off
            src_off += (count + 63) // 64 * 64         # 256-byte aligned float32 blocks
            return o

        def take_dst(nbytes: int) -> int:
            nonlocal dst_off
            o = dst_off
            dst_off += (nbytes + 1023) // 1024 * 1024
            return o

        host_w = []
        for s in range(S):
            layers0 = weights[0][s]
            if len(layers0) != 4:
                raise ValueError("the MLP kernels support exactly 3 hidden layers + 1 output")
            h1, h2, h3 = (int(layers0[k][0].shape[0]) for k in range(3))
            if int(layers0[3][0].shape[0]) != 1:
                raise ValueError("out_dim != 1 is not supported")
            if layers0[0][0].shape[1] != in_dim:
                raise ValueError("first layer width does not match the AEV length")
            self.dims.append((h1, h2, h3))
            W = [[weights[m][s][k][0].detach().to("cpu", torch.float32) for m in range(M)] for k in range(4)]
            if any((weights[m][s][k][1] is None) != (activation == _lib.ACT_GELU) for m in range(M) for k in range(4)):
                raise ValueError("CELU networks need biases in every layer, GELU networks have none")
            Bv = [[torch.zeros(W[k][m].shape[0]) if weights[m][s][k][1] is None
                   else weights[m][s][k][1].detach().to("cpu", torch.float32) for m in range(M)] for k in range(4)]
            for m in range(M):
                if tuple(W[0][m].shape) != (h1, in_dim) or tuple(W[1][m].shape) != (h2, h1) \
                        or tuple(W[2][m].shape) != (h3, h2) or tuple(W[3][m].shape) != (1, h3):
                    raise ValueError("all ensemble members must share the layer widths of an element")
            host_w.append((W, Bv))
            p1, p2, p3 = pad(h1), pad(h2), pad(h3)
            sc = [weight_scale(W[k], self.variant) for k in range(3)]   # one scale per layer, shared by W and W^T
            plan.append(dict(
                h=(h1, h2, h3), p=(p1, p2, p3), sc=sc,
                s_w1=take_src(M * p1 * self.ldx), s_w2=take_src(M * p2 * p1), s_w3=take_src(M * p3 * p2),
                s_b1=take_src(M * p1), s_b2=take_src(M * p2), s_b3=take_src(M * p3), s_w4=take_src(M * p3),
                s_b4=take_src(M),
                d_f1=take_dst(M * p1 * self.ldx * P2), d_f2=take_dst(M * p2 * p1 * P2), d_f3=take_dst(M * p3 * p2 * P2),
                d_b3=take_dst(M * p2 * p3 * P2), d_b2=take_dst(M * p1 * p2 * P2), d_b1=take_dst(self.ldx * M * p1 * P2)))
        host = torch.zeros(src_off, dtype=torch.float32)   # zero weights and biases in the padding:
        for s in range(S):                                   # CELU(0) = 0 meets zero weights: results unchanged
            (W, Bv), q = host_w[s], plan[s]
            (h1, h2, h3), (p1, p2, p3) = q["h"], q["p"]
            w1 = host[q["s_w1"]:q["s_w1"] + M * p1 * self.ldx].view(M, p1, self.ldx)
            w2 = host[q["s_w2"]:q["s_w2"] + M * p2 * p1].view(M, p2, p1)
            w3 = host[q["s_w3"]:q["s_w3"] + M * p3 * p2].view(M, p3, p2)
            b1 = host[q["s_b1"]:q["s_b1"] + M * p1].view(M, p1)
            b2 = host[q["s_b2"]:q["s_b2"] + M * p2].view(M, p2)
            b3 = host[q["s_b3"]:q["s_b3"] + M * p3].view(M, p3)
            w4 = host[q["s_w4"]:q["s_w4"] + M * p3].view(M, p3)
            b4 = host[q["s_b4"]:q["s_b4"] + M]
            for m in range(M):
                if self.col_pad:   # internal column order: radial | col_pad zeros | angular
                    RLc = self.radial_len
                    w1[m, :h1, :RLc] = W[0][m][:, :RLc]
                    w1[m, :h1, RLc + self.col_pad:in_dim + self.col_pad] = W[0][m][:, RLc:]
                else:
                    w1[m, :h1, :in_dim] = W[0][m]
                w2[m, :h2, :h1] = W[1][m]
                w3[m, :h3, :h2] = W[2][m]
                b1[m, :h1], b2[m, :h2], b3[m, :h3] = Bv[0][m], Bv[1][m], Bv[2][m]
                w4[m, :h3] = W[3][m].view(-1)
                b4[m] = Bv[3][m].view(())
        with torch.cuda.device(self.device):
            src = host.pin_memory().to(self.device, non_blocking=True)
            dst = torch.empty(dst_off, dtype=torch.uint8, device=self.device)
            st = torch.cuda.current_stream(self.device).cuda_stream
            L = _lib.lib(self.variant)
            sp0, dp0 = src.data_ptr(), dst.data_ptr()
            for s in range(S):
                q = plan[s]
                (p1, p2, p3), sc = q["p"], q["sc"]
                ldx_ = self.ldx
                jobs = [   # (src, n, k, ld_src, transpose, scale, batch, src stride, dst, dst stride in bytes)
                    (q["s_w1"], p1, ldx_, ldx_, 0, sc[0], M, p1 * ldx_, q["d_f1"], p1 * ldx_ * P2),      # per member [h1][ldx]
                    (q["s_w2"], p2, p1, p1, 0, sc[1], M, p2 * p1, q["d_f2"], p2 * p1 * P2),              # per member [h2][h1]
                    (q["s_w3"], p3, p2, p2, 0, sc[2], M, p3 * p2, q["d_f3"], p3 * p2 * P2),              # per member [h3][h2]
                    (q["s_w3"], p2, p3, p2, 1, sc[2], M, p3 * p2, q["d_b3"], p2 * p3 * P2),              # W3^T [h2][h3]
                    (q["s_w2"], p1, p2, p1, 1, sc[1], M, p2 * p1, q["d_b2"], p1 * p2 * P2),              # W2^T [h1][h2]
                    (q["s_w1"], ldx_, M * p1, ldx_, 1, sc[0], 1, 0, q["d_b1"], 0),                       # W1^T [ldx][M*h1]
                ]
                for (so, n_, k_, ld_, tr, scale, batch, sstr, do, dstr) in jobs:
                    check(L.ani_b200_pack_b_operand(sp0 + 4 * so, n_, k_, ld_, tr, scale, batch, sstr, dp0 + do, dstr, st),
                          "pack_b_operand")
                spm = mdl.sp[s]
                spm.h1, spm.h2, spm.h3 = p1, p2, p3
                for k in range(3):
                    spm.w_scale[k] = sc[k]
                spm.w_scale[3] = 1.0
                for name, off in (("b1", q["s_b1"]), ("b2", q["s_b2"]), ("b3", q["s_b3"]), ("w4", q["s_w4"]),
                                  ("b4", q["s_b4"])):
                    setattr(spm, name, sp0 + 4 * off)
                for name, off in (("t_f1", q["d_f1"]), ("t_f2", q["d_f2"]), ("t_f3", q["d_f3"]), ("t_b3", q["d_b3"]),
                                  ("t_b2", q["d_b2"]), ("t_b1", q["d_b1"])):
                    setattr(spm, name, dp0 + off)
        # scratch of the per-step compaction of the layer-1 backward operands (live AEV column blocks only; as large
        # as those operands together; ani_mlp_model::b1_compact)
        b1c = torch.empty(sum(self.ldx * (M * q["p"][0] // 32) * 32 * P2 for q in plan), dtype=torch.uint8,
                          device=self.device)
        mdl.b1_compact = b1c.data_ptr()
        self._keep = [src, dst, b1c]
        self._plan = plan
        # the plain fp32 weights next to the tiled operands (W1 in the internal column order), which the Hessian's
        # tangent network pass reads (Engine.hessian)
        self.plain_weights = _lib.HessianWeights()
        for s in range(S):
            q = plan[s]
            self.plain_weights.w1[s] = sp0 + 4 * q["s_w1"]
            self.plain_weights.w2[s] = sp0 + 4 * q["s_w2"]
            self.plain_weights.w3[s] = sp0 + 4 * q["s_w3"]
        mdl.h1_max = max(q["p"][0] for q in plan)
        mdl.h2_max = max(q["p"][1] for q in plan)
        mdl.h3_max = max(q["p"][2] for q in plan)
        self.set_active_members(list(range(M)))

    def set_active_members(self, idxs: tp.Sequence[int]) -> None:
        """nn/_core.py:99-110: the ensemble output is the mean over the active members."""
        for i in idxs:
            if not 0 <= i < self.num_members:
                raise IndexError(f"Idx {i} should be 0 <= idx < {self.num_members}")
        self.active = list(idxs)
        # captured CUDA graphs bake the member scales in: they are keyed by this tuple (Engine.run)
        self.active_key = tuple(self.active)
        for m in range(_lib.ANI_MAX_MEMBERS):
            self.model.member_scale[m] = (1.0 / len(self.active)) if m in self.active else 0.0

    @property
    def ld(self) -> tp.Tuple[int, int, int]:
        M = self.num_members
        return M * self.model.h1_max, M * self.model.h2_max, M * self.model.h3_max

    @property
    def act_cols(self) -> tp.Tuple[int, int, int]:
        """Columns of the act1 / act2 / act3 buffers: ``ld``, with room for the derivative operand of a GELU model
        directly behind the activation operands act1 / act2 (include/ani_b200.h section 6)."""
        ld1, ld2, ld3 = self.ld
        k = 2 if self.activation == _lib.ACT_GELU else 1
        return k * ld1, k * ld2, ld3

    def flops_per_atom(self, species_index: int, backward: bool = True) -> float:
        h1, h2, h3 = self.dims[species_index]
        macs = self.in_dim * h1 + h1 * h2 + h2 * h3 + h3
        return 2.0 * macs * self.num_members * (2 if backward else 1)


class Workspace:
    """All device buffers for one (n_conf, n_per_conf) problem shape."""

    def __init__(self, n_conf: int, n_per_conf: int, num_species: int, ldx: int, ld: tp.Tuple[int, int, int],
                 num_members: int, nbr_cap: int, device: torch.device, owned_cap: tp.Optional[int] = None,
                 variant: tp.Optional[str] = None):
        n = n_conf * n_per_conf
        self.n, self.n_conf, self.n_per_conf = n, n_conf, n_per_conf
        owned = n if owned_cap is None else min(n, owned_cap)
        self.rows_cap = (owned + num_species * (TILE - 1) + TILE - 1) // TILE * TILE
        self.max_bins = max(64, n + 2) if n_conf == 1 else n_conf + 2
        i32 = dict(dtype=torch.int32, device=device)
        f32 = dict(dtype=torch.float32, device=device)
        self.grid = torch.zeros(C.sizeof(Grid) // 4, **i32)
        # What a host-driven loop moves per step lives in TWO contiguous blocks, so that calculator.HostCalculator needs one
        # H2D and one D2H copy (each copy is a node of the captured graph with its own DMA set-up latency):
        #   in_block  f32: [cell 9 x n_conf (one per conformer, or the shared one first) | pad to 16 | coords 3 n]
        #   out_block u8 : [energies f64 x n_conf | status i32 | pad to 16 B | grad f32 x 3 n]
        # followed, in the same allocation (out_full), by what the query-by-committee step adds (Engine.run(...,
        # members=True)), so that it too needs one D2H copy while the ordinary step still copies out_block only:
        #   [member energies f64 x M x n_conf | qbc f64 x n_conf | pad to 16 B | atom stats f32 x 3 n]
        # and then by what a step with charges adds (Engine.run(..., charges=True), calculator.calculate_with_charges):
        #   [pad to 16 B | dipoles f64 x 3 n_conf | charges f32 x n]
        self.in_coords_off = (9 * n_conf + 15) // 16 * 16
        self.in_block = torch.zeros(self.in_coords_off + 3 * n, **f32)
        self._out_grad_off = (8 * n_conf + 4 + 15) // 16 * 16
        out_len = self._out_grad_off + 12 * n
        self._out_qbc_off = (out_len + 15) // 16 * 16
        self._out_stats_off = (self._out_qbc_off + 8 * (num_members + 1) * n_conf + 15) // 16 * 16
        self._out_chg_off = (self._out_stats_off + 12 * n + 15) // 16 * 16
        self.out_full = torch.zeros(self._out_chg_off + 24 * n_conf + 4 * n, dtype=torch.uint8, device=device)
        self.out_block = self.out_full[:out_len]
        self.member_energies = self.out_full[self._out_qbc_off:self._out_qbc_off + 8 * num_members * n_conf].view(
            torch.float64).view(num_members, n_conf)
        self.qbc = self.out_full[self._out_qbc_off + 8 * num_members * n_conf:
                                 self._out_qbc_off + 8 * (num_members + 1) * n_conf].view(torch.float64)
        self.atom_stats = self.out_full[self._out_stats_off:self._out_stats_off + 12 * n].view(torch.float32).view(3, n)
        self.dipoles = self.out_full[self._out_chg_off:self._out_chg_off + 24 * n_conf].view(torch.float64).view(n_conf, 3)
        self.charges = self.out_full[self._out_chg_off + 24 * n_conf:].view(torch.float32)
        # the charge networks' own activations and raw outputs (one member), allocated on the first step with charges
        # (Engine.charge_buffers): the energy networks' act1..act3 / e_member are live until the energy reduction
        self.q_act: tp.Optional[tp.Tuple[Tensor, Tensor, Tensor]] = None
        self.q_raw: tp.Optional[Tensor] = None
        # per-member dE/dAEV slabs f32[M][rows_cap][ldx] and dE_m/dcoords f32[M][n][3] of the query-by-committee step:
        # allocated on its first use (Engine.members_buffers; at 10 k atoms the slabs of 8 members take ~340 MB)
        self.dx_members: tp.Optional[Tensor] = None
        self.grad_members: tp.Optional[Tensor] = None
        self.status = self.out_block[8 * n_conf: 8 * n_conf + 4].view(torch.int32)
        self.bin_start = torch.zeros(self.max_bins + 2, **i32)
        self.sorted_orig = torch.zeros(n, **i32)
        self.orig_to_sorted = torch.zeros(n, **i32)
        self.spos = torch.zeros(n, 4, **f32)
        self.sbin = torch.zeros(n, **i32)
        self.scratch = torch.zeros(3 * n + self.max_bins + 2 + (n // 256 + 3) * 8 + 64, **i32)
        self.row_of = torch.zeros(n, **i32)
        self.row_atom = torch.zeros(self.rows_cap, **i32)
        self.tile_species = torch.zeros(self.rows_cap // TILE, **i32)
        self.layout_info = torch.zeros(16, **i32)
        self.aev_blocks = torch.zeros(ldx // 32 + 3, **i32)   # [count, ids..., element mask, changed flag]
        self.n_blocks = ldx // 32
        self.bucket_ranges = torch.zeros((self.max_bins - 1) * 27 * 8, **f32) if n_conf == 1 else None
        # per-bucket species offsets (ani_b200_prepare_step -> ani_b200_aev_forward): i32[max_bins][8].  Experiment
        # (ANI_B200_AEV_BSS=1): lets the AEV forward skip its candidate-counting pass at the price of one more dependent
        # global load at the head of every CTA; off by default
        self.bucket_species = (torch.zeros(self.max_bins * 8, **i32)
                               if n_conf == 1 and os.environ.get("ANI_B200_AEV_BSS", "0") != "0" else None)
        self.nbr_cap = nbr_cap
        self.nbr_cnt = torch.zeros(n, **i32)
        self.nbr_list = torch.zeros(n * nbr_cap, **i32)
        # x / act*: "tiled operand" form (16-bit pieces of every value); dx: plain float32 rows
        self.x = operand_buffer(self.rows_cap, ldx, device, variant)
        self.dx = torch.zeros(self.rows_cap, ldx, **f32)
        self.act1 = operand_buffer(self.rows_cap, ld[0], device, variant)
        self.act2 = operand_buffer(self.rows_cap, ld[1], device, variant)
        self.act3 = operand_buffer(self.rows_cap, ld[2], device, variant)
        self.e_member = torch.zeros(num_members, self.rows_cap, **f32)
        self.mlp_sync = torch.zeros(6 * (self.rows_cap // TILE) * _lib.ANI_MAX_MEMBERS + 8, **i32)   # ani_b200_mlp_step counters
        self.species_i32 = torch.zeros(n, **i32)
        self.coords = self.in_block[self.in_coords_off:].view(n, 3)
        self.cell = self.in_block[:9]
        self.cells = self.in_block[:9 * n_conf].view(n_conf, 9)   # grid mode 3: one cell per conformer
        self.grad = self.out_block[self._out_grad_off:].view(torch.float32).view(n, 3)
        self.atomic = torch.zeros(n, **f32)
        self.member_atomic = torch.zeros(num_members, n, **f32)
        self.energies = self.out_block[:8 * n_conf].view(torch.float64)
        # where the step's kernels ACCUMULATE forces / conformer energies: these buffers, or -- multi-GPU,
        # parallel.ShardedEngine.attach -- partial-sum buffers in peer-mapped memory whose reduction over the
        # ranks (reducer.launch, the last launch of the step) lands in `grad` / `energies`
        self.grad_ptr = self.grad.data_ptr()
        self.energies_ptr = self.energies.data_ptr()
        self.reducer: tp.Any = None
        # distinct elements seen at graph-capture time (0 = not known): sizes the shared-memory gradient
        # table of the AEV backward kernel; the results never depend on it (Engine.note_composition)
        self.max_elements = 0
        # Verlet-skin reuse of the bucket grid (Engine.skin > 0): binned positions, wrapping lattice
        # vectors and the "an atom left its skin/2 sphere" word (ani_b200_verlet_positions)
        self.ref_pos = torch.zeros(n, 4, **f32)
        self.ref_shift = torch.zeros(n, 4, **f32)
        self.moved = torch.zeros(1, **i32)
        # partial sums of the virial W_ab = sum_pairs (dE/dDelta)_a Delta_b (ani_b200_aev_backward)
        self.virial = torch.zeros(_lib.ANI_VIRIAL_SLOTS, 9, dtype=torch.float64, device=device)
        self.periodic = n_conf == 1
        self.lattice: tp.Optional[Tensor] = None
        self._retired: tp.List[Tensor] = []

    def make_periodic(self) -> None:
        """Size the bucket buffers of a batch for periodic cells (grid modes 2 and 3), once, on its first use with a
        cell: every conformer gets the bucket capacity of a single-system workspace of its atoms, so that its sub-grid
        is the grid a single system would get.  The buffers of the open batch (one bucket per conformer) stay alive
        for the CUDA graphs captured with them."""
        if self.periodic:
            return
        n, dev = self.n, self.grid.device
        i32 = dict(dtype=torch.int32, device=dev)
        self._retired += [self.bin_start, self.scratch]
        self.max_bins = self.n_conf * (max(64, self.n_per_conf + 2) - 1) + 1
        self.bin_start = torch.zeros(self.max_bins + 2, **i32)
        self.scratch = torch.zeros(3 * n + self.max_bins + 2 + (n // 256 + 3) * 8 + 64, **i32)
        self.bucket_ranges = torch.zeros((self.max_bins - 1) * 27 * 8, dtype=torch.float32, device=dev)
        self.bucket_species = (torch.zeros(self.max_bins * 8, **i32)
                               if os.environ.get("ANI_B200_AEV_BSS", "0") != "0" else None)
        self.virial = torch.zeros(self.n_conf * _lib.ANI_VIRIAL_SLOTS, 9, dtype=torch.float64, device=dev)
        # grid mode 3: per conformer {cell, inverse}, written by the preparation of every step
        self.lattice = torch.zeros(self.n_conf, _lib.ANI_LATTICE_STRIDE, dtype=torch.float32, device=dev)
        self.periodic = True


def _grid_mode(n_conf: int, pbc: bool, conformer_cells: bool = False) -> int:
    """ani_grid::mode: 0 one system, 1 an open batch (one bucket per conformer), 2 a periodic batch in one shared cell
    (one sub-grid per conformer), 3 a periodic batch with one cell per conformer."""
    if conformer_cells and n_conf > 1:
        return 3
    return 0 if n_conf == 1 else (2 if pbc else 1)


def conformer_cells(cell: tp.Optional[Tensor], n_conf: int) -> bool:
    """True if ``cell`` is one cell per conformer, (C, 3, 3) (grid mode 3); False for one shared (3, 3) cell or None."""
    if cell is None or cell.dim() == 2:
        return False
    if cell.shape != (n_conf, 3, 3):
        raise ValueError(f"cell must be (3, 3) or one cell per conformer, ({n_conf}, 3, 3); got {tuple(cell.shape)}")
    return True


def check_pair_cutoff(cutoff: float, rcr: float) -> None:
    """A pair potential runs in the fused step over the neighbour words of the AEV forward, which hold nothing beyond
    the radial cutoff: its own cutoff may not be larger (there is no second neighbour search)."""
    if not _f32(cutoff) <= _f32(rcr):
        raise ValueError(f"a pair potential of the fused step needs cutoff <= the radial AEV cutoff ({rcr} A), got "
                         f"{cutoff}: it is evaluated over the AEV's neighbour list, which holds nothing beyond it")


# Jacobian rows (3 per neighbour word) of one chunk of central atoms in Engine.hessian: at ldx = 1024 and ANI-2x widths,
# 32 768 rows take about 130 MB of Jacobian and 130 MB of tangent scratch
HESSIAN_ROW_BUDGET = 32768


class _HessianPlan(tp.NamedTuple):
    """One chunk of central atoms of Engine.hessian, in the layout of ani_hessian_chunk (include/ani_b200.h
    section 9)."""
    atom: np.ndarray          # i32 [n_slots] sorted index
    row_off: np.ndarray       # i32 [n_slots]
    row_slot: np.ndarray      # i32 [rows]
    tile_species: np.ndarray  # i32 [rows / ANI_HESSIAN_ROW_ALIGN]
    block_off: np.ndarray     # i64 [n_slots]
    rows: int
    block_floats: int
    max_count: int


def _hessian_chunks(cnt: np.ndarray, species: np.ndarray, row_budget: int) -> tp.Iterator[_HessianPlan]:
    """Split the real sorted atoms (neighbour counts ``cnt``, element indices ``species``) into chunks whose Jacobian
    rows, species segments aligned to ANI_HESSIAN_ROW_ALIGN, fit ``row_budget`` (a chunk holds at least one atom)."""
    align = _lib.ANI_HESSIAN_ROW_ALIGN
    if row_budget < align:
        raise ValueError(f"row_budget must be at least {align}")
    up = lambda v: (v + align - 1) // align * align  # noqa: E731
    order = np.argsort(species, kind="stable")
    chunk: tp.List[int] = []
    seg: tp.Dict[int, int] = {}

    def plan(atoms: tp.List[int]) -> _HessianPlan:
        atom = np.asarray(atoms, dtype=np.int32)   # species-major (``order``)
        row_off = np.zeros(len(atom), dtype=np.int32)
        block_off = np.zeros(len(atom), dtype=np.int64)
        slots, tiles = [], []
        r, b, prev = 0, 0, None
        for k, a in enumerate(atom):
            s = int(species[a])
            if s != prev and prev is not None:
                pad = up(r) - r
                slots.append(np.full(pad, -1, dtype=np.int32))
                r += pad
            if s != prev:
                tiles.append((r // align, s))
            prev = s
            row_off[k], block_off[k] = r, b
            m3 = 3 * int(cnt[a])
            slots.append(np.full(m3, k, dtype=np.int32))
            r += m3
            b += m3 * m3
        pad = up(max(r, 1)) - r
        slots.append(np.full(pad, -1, dtype=np.int32))
        rows = r + pad
        tile_species = np.zeros(rows // align, dtype=np.int32)
        for t0, s in tiles:
            tile_species[t0:] = s
        return _HessianPlan(atom, row_off, np.concatenate(slots), tile_species, block_off, rows, max(b, 1),
                            int(cnt[atom].max()))

    for a in order:
        s, m3 = int(species[a]), 3 * int(cnt[a])
        grown = dict(seg)
        grown[s] = grown.get(s, 0) + m3
        if chunk and sum(up(v) for v in grown.values()) > row_budget:
            yield plan(chunk)
            chunk, grown = [], {s: m3}
        chunk.append(int(a))
        seg = grown
    if chunk:
        yield plan(chunk)


class StepResult(tp.NamedTuple):
    energies: Tensor          # (C,) float64: NN energy + self energies of the owned atoms
    atomic_energies: Tensor   # (C, A) float32: NN atomic energies (ensemble mean), 0 for padding
    member_atomic: Tensor     # (M, C, A) float32 per-member NN atomic energies
    grad: tp.Optional[Tensor]  # (C, A, 3) float32 dE/dcoords (forces = -grad) or None
    virial: tp.Optional[Tensor] = None  # (3, 3) float64 sum_pairs (dE/dDelta)_a Delta_b (stress = virial / volume);
    #                                     (C, 3, 3) for a periodic batch


class MembersResult(tp.NamedTuple):
    """What the query-by-committee step (``Engine.run(..., members=True)``) adds; member k is ``nets.active[k]``."""
    energies: Tensor           # (M_active, C) float64: member energies incl. self energies
    grad: Tensor               # (M_active, C, A, 3) float32: dE_m/dcoords
    qbc: Tensor                # (C,) float64: std_m(E_m) / sqrt(real atoms), arch.py:439-485
    force_magnitudes: Tensor   # (C, A) float32: mean_m |F_m|, arch.py:510-540
    force_relative_stdev: Tensor   # (C, A) float32: (std_m |F_m| + 1e-8) / (mean + 1e-8), arch.py:543-576
    force_relative_range: Tensor   # (C, A) float32: (max_m |F_m| - min_m |F_m| + 1e-8) / (mean + 1e-8)


class ChargeParams(tp.NamedTuple):
    """The normaliser and dipole parameters of a charge model (the host arguments of ``ani_b200_charges``)."""
    weights: tp.Tuple[float, ...]        # per element (ChargeNormalizer.weights); unused without ``normalize``
    scale_by_q2: bool = False            # ChargeNormalizer.scale_weights_by_charges_squared
    normalize: bool = True               # False: BaseChargeNormalizer (raw charges)
    masses: tp.Optional[tp.Tuple[float, ...]] = None   # per element; needed for the centre-of-mass frame only
    frame: int = 2                       # dipole reference point: 0 centre of mass, 1 centre of geometry, 2 origin

    def arrays(self) -> tp.Tuple[tp.Any, tp.Any]:
        w = (C.c_float * len(self.weights))(*self.weights)
        m = None if self.masses is None else (C.c_float * len(self.masses))(*self.masses)
        return w, m


class ChargesResult(tp.NamedTuple):
    """What a step with charges (``Engine.run(..., charges=True)``) adds."""
    charges: Tensor    # (C, A) float32: normalised atomic charges (e), 0 for padding
    dipoles: Tensor    # (C, 3) float64: sum_i q_i (r_i - r_ref) (e * Angstrom)


class Engine:
    """Fused ANI energy(+force) step on one GPU.  ``lo_frac/hi_frac`` select the slice of
    bucket-sorted atoms this engine owns (multi-GPU sharding, see parallel.py)."""

    def __init__(self, consts: AEVConstants, nets: PackedNetworks, sae: tp.Optional[tp.Sequence[float]] = None,
                 nbr_cap: int = 128, cuda_graph: bool = True, pairs: tp.Sequence[PairParams] = (),
                 dispersion: tp.Optional[tp.Tuple[D3Params, Tensor]] = None,
                 charges: tp.Optional[tp.Tuple[PackedNetworks, ChargeParams]] = None):
        """``pairs``: the ``ani_pair_params`` of the model's pair potentials (potentials.PairPotential.params()); each
        adds one launch to the step, a model without any issues exactly the launches it issued before.  The repulsion
        kinds (0 xTB, 1 ZBL) run over the AEV's neighbour words and need cutoff <= Rcr (``_pair_potentials``); the LJ
        and Coulomb kinds (2-6) run over a neighbour search of their own cutoff, at any cutoff (``_search_pairs``).  ``dispersion``: the ``ani_d3_params`` and device tables of a D3 term
        (potentials.TwoBodyDispersionD3.params() / .tables(device)), or None; it adds three launches to a step with
        forces and two to one without (``_dispersion``).  ``charges``: the packed charge networks (one member) and the
        normaliser / dipole parameters of a charge model; a step asked for charges (``run(..., charges=True)``) runs
        them forward-only on the step's AEVs and adds the launches of ``_charge_pass``, any other step is unchanged."""
        if nets.in_dim != consts.out_dim:
            raise ValueError("network input width != AEV length")
        if nets.num_species != consts.num_species:
            raise ValueError("network / AEV species mismatch")
        self.consts, self.nets = consts, nets
        for p in pairs:
            if p.kind in (0, 1):
                check_pair_cutoff(math.inf if p.cutoff_fn == 2 else p.cutoff, consts.rcr)
            if p.num_species != consts.num_species:
                raise ValueError("pair potential / AEV species mismatch")
        self.pairs = [p for p in pairs if p.kind in (0, 1)]
        self.search_pairs = [p for p in pairs if p.kind not in (0, 1)]
        if dispersion is not None:
            d3p, d3t = dispersion
            if d3p.cutoff_fn == 2 or not d3p.cutoff > 0:
                raise ValueError("D3 in the fused step needs a finite cutoff (its neighbour search runs on the grid)")
            if d3p.num_species != consts.num_species:
                raise ValueError("D3 / AEV species mismatch")
            if d3t.device != nets.device or d3t.dtype != torch.float32 or d3t.numel() != d3p.num_species ** 2 * 100:
                raise ValueError("D3 tables must be float32 (S, S, 25, 4) on the engine's device")
        self.dispersion = dispersion
        self.charges: tp.Optional[tp.Tuple[PackedNetworks, ChargeParams]] = None
        self.set_charges(charges)
        self.device = nets.device
        self.params = consts.to_struct()
        # internal column order of the tiled AEV operand / dE/dAEV rows: must be the one the layer-1 weights were packed in
        if nets.col_pad and nets.radial_len != consts.num_species * len(consts.shf_r):
            raise ValueError("the networks were packed for another radial AEV length")
        self.params.ang_pad = nets.col_pad
        self.nbr_cap = nbr_cap
        # > 0: buckets are built for cutoff + skin, so that a grid can be reused while no atom has moved
        # more than skin/2 (run(..., reuse=True); calculator.HostCalculator drives it)
        self.skin = 0.0
        self.sae = None
        if sae is not None:
            self.sae = torch.tensor(list(sae), dtype=torch.float64, device=self.device)
        self._ws: tp.Dict[tp.Tuple[int, int], Workspace] = {}
        self.cuda_graph = cuda_graph
        self.graph_after = 3   # eager launches of a problem shape before its CUDA graph is captured
        self._graphs: tp.Dict[tp.Any, torch.cuda.CUDAGraph] = {}   # insertion order = LRU order
        self.max_graphs = 16
        self._graph_seen: tp.Dict[tp.Any, int] = {}
        self.variant = nets.variant
        self.lib = _lib.lib(self.variant)
        self.launches_per_step = 0
        # The forward-only pass of the charge networks: "step" = ani_b200_mlp_step(..., want_backward=0) (one data-flow
        # launch per window), "chained" = ani_b200_mlp_forward (three launches of the GEMM kernel).  On the H100 the
        # data-flow form was 2-3 % faster at water 10 k and on the GDB batch of 256 (tools/charge_timing.py, DESIGN §4.8)
        self.charge_mlp = os.environ.get("ANI_B200_CHARGE_MLP", "step")
        # per-stage CUDA-event timing (bench.py's roofline leg); off by default
        self.profile = False
        # zero-fill of dE/dAEV and the energy reduction on a forked side stream (see _launch); off by default --
        # inside the graph the two kernels cost little more than their dependency edges
        self.side_stream = os.environ.get("ANI_B200_SIDE_STREAM", "0") != "0"
        self.overlap_reduce = os.environ.get("ANI_B200_OVERLAP_REDUCE", "1") != "0"
        # The MLP of a step: ONE persistent data-flow launch or the six chained launches of the same GEMM kernel
        # (csrc/gemm_tc.cuh).  The data-flow list avoids the launch boundaries and the per-launch tile-count quantisation;
        # on the H100 it is as fast or faster from one wave of units per layer up (water 10 k, 50 k-atom protein, GDB
        # batch of 256), while below a wave (water 1 k) the chained launches are as fast and hand a row tile over
        # without an L2 counter.  "auto" applies that rule; ANI_B200_MLP_FUSED=0 / 1 forces one of them.
        self.mlp_mode = os.environ.get("ANI_B200_MLP_FUSED", "auto")
        # Where "auto" picks the data-flow launch and gradients are wanted, one launch of resident chains
        # (csrc/mlp_resident.cuh) replaces it: every intermediate of a (row tile, member) chain stays in shared
        # memory.  It exists in the 2 x fp16 build for hidden widths up to 256 (ani_b200_mlp_step_resident).
        m = nets.model
        self._resident_ok = (_lib.operand_format(self.variant).parts == 2
                             and max(m.h1_max, m.h2_max, m.h3_max) <= 256)
        self.mlp_resident = False
        self._num_sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        self._side_stream: tp.Optional[torch.cuda.Stream] = None
        self._ev: tp.List[torch.cuda.Event] = []
        self.stage_events: tp.Dict[str, tp.List[tp.Tuple[torch.cuda.Event, torch.cuda.Event]]] = {}
        self.hessian_count = 0   # Hessians computed by this engine (``hessian``)

    def _timed(self, name: str, fn: tp.Callable[[], int]) -> None:
        """Run one C-ABI stage; with ``profile`` on, bracket it with events on the launch stream."""
        if not self.profile:
            check(fn(), name)
            return
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        check(fn(), name)
        b.record()
        self.stage_events.setdefault(name, []).append((a, b))

    def stage_times_ms(self) -> tp.Dict[str, float]:
        """Mean device time per call of every stage (synchronises)."""
        torch.cuda.synchronize(self.device)
        return {k: sum(a.elapsed_time(b) for a, b in v) / len(v) for k, v in self.stage_events.items() if v}

    # -- workspaces ------------------------------------------------------------------------
    def workspace(self, n_conf: int, n_per_conf: int) -> Workspace:
        key = (n_conf, n_per_conf)
        ws = self._ws.get(key)
        if ws is None:
            ws = self.new_workspace(n_conf, n_per_conf)
            self._ws[key] = ws
        return ws

    def new_workspace(self, n_conf: int, n_per_conf: int) -> Workspace:
        """A workspace of this shape that the engine does not cache, for a caller that keeps state in it from one step
        to the next (md: the forces of the current positions); run it through ``_launch``, whose captured graphs are
        the caller's (``run`` keys its graphs by shape, not by workspace)."""
        ws = Workspace(n_conf, n_per_conf, self.consts.num_species, self.nets.ldx, self.nets.act_cols,
                       self.nets.num_members, self.nbr_cap, self.device, variant=self.variant)
        if self.dispersion is not None:   # coordination numbers and dE/dCN of every atom (D3 scratch)
            ws.d3_cn = torch.zeros(ws.n, dtype=torch.float32, device=self.device)
            ws.d3_dedcn = torch.zeros(ws.n, dtype=torch.float32, device=self.device)
        return ws

    def _stage_inputs(self, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor], pbc: bool
                      ) -> tp.Tuple[Workspace, bool]:
        """Copy a step's inputs into the persistent buffers of its workspace (what a captured graph reads).  Returns the
        workspace and whether it holds one cell per conformer."""
        n_conf, n_per_conf = species.shape
        if coords.shape != (n_conf, n_per_conf, 3):
            raise ValueError("coords must have shape (C, A, 3)")
        if pbc and cell is None:
            raise ValueError("If pbc is not None, cell should be present")
        per_conf = bool(pbc) and conformer_cells(cell, n_conf)
        if per_conf and n_conf == 1:
            cell, per_conf = cell[0], False   # one conformer: its cell is the shared cell
        ws = self.workspace(n_conf, n_per_conf)
        if pbc:
            ws.make_periodic()
        ws.species_i32.copy_(species.reshape(-1))
        ws.coords.copy_(coords.reshape(-1, 3))
        if per_conf:
            ws.cells.copy_(cell.reshape(n_conf, 9))
        elif pbc:
            ws.cell.copy_(cell.reshape(-1))
        return ws, per_conf

    # -- one step --------------------------------------------------------------------------
    def step(self, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None, pbc: bool = False,
             want_grad: bool = True, shard: tp.Tuple[int, int] = (0, 1), want_virial: bool = False,
             check: bool = False, want_charges: bool = False) -> StepResult:
        """species (C, A) int (element indices, -1 padding), coords (C, A, 3) on this device.
        ``shard = (rank, world)``: only atoms whose bucket-sorted position falls into this
        rank's slice are evaluated; gradients/energies are partial sums to be all-reduced.

        The launch sequence of a given problem shape is captured into a CUDA graph on its fourth
        use and replayed afterwards (``cuda_graph=False`` at construction disables this)."""
        dev = self.device
        if species.device != dev or coords.device != dev:
            raise ValueError(f"inputs must live on {dev} (the engine has no CPU path)")
        ws, per_conf = self._stage_inputs(species, coords, cell, pbc)
        res = self.run(ws, bool(pbc), want_grad, shard, want_virial=want_virial, conformer_cells=per_conf,
                       charges=want_charges)
        if check:   # one 4-byte D2H read: cell too small / neighbour overflow / operand range raise here
            self.check_status(ws)
        return res

    def run(self, ws: Workspace, pbc: bool, want_grad: bool = True, shard: tp.Tuple[int, int] = (0, 1),
            reuse: bool = False, want_virial: bool = False, conformer_cells: bool = False,
            members: bool = False, charges: bool = False) -> StepResult:
        """One step on inputs that are ALREADY in the workspace buffers (``ws.species_i32``,
        ``ws.coords``, ``ws.cell`` -- or, with ``conformer_cells``, one cell per conformer in ``ws.cells``) -- the
        entry point of host-driven loops that copy straight into them (calculator.HostCalculator).  The results alias
        workspace buffers.

        ``members=True``: the query-by-committee step (``_launch_members``).  Besides the ordinary results (the
        gradient is the mean of the members' gradients) it leaves every active member's energy and gradient and the
        force / energy disagreement statistics in the workspace (``members_result``).  One GPU only.

        ``charges=True`` (an engine built with ``charges``): the step also leaves the normalised atomic charges and the
        dipoles in the workspace (``charges_result``).  One GPU only, not in the query-by-committee step: the
        normaliser needs every atom's raw charge."""
        n, n_conf, n_per_conf = ws.n, ws.n_conf, ws.n_per_conf
        members = bool(members)
        charges = bool(charges)
        if charges:
            if self.charges is None:
                raise ValueError("this engine has no charge networks")
            if members or tuple(shard) != (0, 1) or ws.reducer is not None:
                raise ValueError("charges are computed unsharded and outside the query-by-committee step: the "
                                 "normaliser needs every atom's raw charge")
            self.charge_buffers(ws)
        if members and (tuple(shard) != (0, 1) or not want_grad or want_virial):
            raise ValueError("the query-by-committee step runs unsharded, with forces and without the virial")
        rank, world = shard
        lo = (n * rank) // world
        hi = (n * (rank + 1)) // world
        periodic_batch = bool(pbc) and n_conf > 1
        conformer_cells = bool(conformer_cells)
        if conformer_cells and not periodic_batch:
            raise ValueError("one cell per conformer needs a periodic batch (C > 1, pbc)")
        if want_virial and (not want_grad or reuse or (n_conf != 1 and not periodic_batch)):
            raise ValueError("the virial comes out of the force pass of a single system or a periodic batch with a "
                             "freshly built grid")
        if periodic_batch and not ws.periodic:
            raise ValueError("the workspace of a periodic batch needs Workspace.make_periodic() first")
        if periodic_batch and reuse:
            raise ValueError("reuse=True (Verlet skin) is not supported for periodic batches")
        self.check_pair_cutoffs(pbc)
        key = (n_conf, n_per_conf, bool(pbc), bool(want_grad), lo, hi, self.nets.active_key, bool(reuse), self.skin,
               bool(want_virial), self.mlp_mode, conformer_cells, members, tuple(p.kind for p in self.search_pairs))
        if charges:   # (the charge networks' operands and the normaliser / dipole parameters are baked into the capture)
            key = key + (self.charges[0], self.charges[1], self.charge_mlp)
        if reuse and not self.skin > 0:
            raise ValueError("reuse=True needs Engine.skin > 0 and a previous step that built the grid")
        if members:
            self.members_buffers(ws)
        with torch.cuda.device(self.device):   # the C-ABI launches on the CURRENT device's stream
            if not self.cuda_graph or self.profile:
                self._launch(ws, bool(pbc), want_grad, lo, hi, reuse, want_virial, conformer_cells, members, charges)
            else:
                graph = self._graphs.get(key)
                if graph is not None:
                    self._graphs[key] = self._graphs.pop(key)   # most recently used last
                    graph.replay()
                elif self._graph_seen.get(key, 0) < self.graph_after:
                    # the first few uses of a shape run eagerly (one-off shapes never pay for a capture)
                    if len(self._graph_seen) > 4 * self.max_graphs:
                        self._graph_seen.clear()
                    self._graph_seen[key] = self._graph_seen.get(key, 0) + 1
                    self._launch(ws, bool(pbc), want_grad, lo, hi, reuse, want_virial, conformer_cells, members, charges)
                else:
                    self.note_composition(ws)
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        self._launch(ws, bool(pbc), want_grad, lo, hi, reuse, want_virial, conformer_cells, members, charges)
                    while len(self._graphs) >= self.max_graphs:   # evict the least recently used capture
                        self._graphs.pop(next(iter(self._graphs)))
                    self._graphs[key] = graph
                    graph.replay()
        # kernels launched by this library in one step (memsets excluded):
        # prepare 1 (+1 grid kernel for open single systems), AEV fwd 1, GEMM fwd 3,
        # (zero + GEMM bwd 3 + AEV bwd 1), reduce 1; the fused MLP: zero + one launch (resident chains) or + one per
        # window (data flow)
        if members:
            # the resident launch (+ its operand gather) or one data-flow launch per window (want_backward=2), then the
            # members' AEV backward and the two statistics launches
            mlp = (2 if self._use_resident_mlp(n, True) else
                   self.lib.ani_b200_mlp_step_windows(C.byref(self.nets.model), ws.rows_cap)) + 2
        elif self._use_resident_mlp(hi - lo, want_grad):
            mlp = 2
        elif self._use_dataflow_mlp(hi - lo):
            mlp = self.lib.ani_b200_mlp_step_windows(C.byref(self.nets.model), ws.rows_cap) + (1 if want_grad else 0)
        else:
            mlp = 3 + (4 if want_grad else 0)
        self.launches_per_step = (1 + (0 if (pbc or n_conf > 1) else 1) + 1 + mlp + (1 if want_grad else 0) + 1
                                  + len(self.pairs) + len(self.search_pairs))
        if self.dispersion is not None:   # CN, energies + dE/dCN, and the chain where forces are wanted
            self.launches_per_step += 3 if (want_grad or members) else 2
        if charges:
            self.launches_per_step += self._charge_launches(ws)
        # what the workspace now holds, for Engine.hessian: (periodic, dE/dAEV rows written, sharded)
        ws.last_run = (bool(pbc), bool(want_grad) and not members, (lo, hi) != (0, n) or ws.reducer is not None)
        grad = ws.grad.view(n_conf, n_per_conf, 3) if want_grad else None
        virial = None
        if want_virial:
            virial = ws.virial.view(n_conf, -1, 9).sum(1).view(n_conf, 3, 3)
            if n_conf == 1:
                virial = virial[0]
        return StepResult(ws.energies, ws.atomic.view(n_conf, n_per_conf),
                          ws.member_atomic.view(-1, n_conf, n_per_conf), grad, virial)

    def check_pair_cutoffs(self, pbc: bool) -> None:
        if pbc and any(p.cutoff_fn == 2 for p in self.search_pairs):
            raise ValueError("PBC can't use an infinite cutoff: a pair potential without a cutoff runs on open systems "
                             "only")

    def _prepare(self, ws: Workspace, pbc: bool, conformer_cells: bool, lo: int, hi: int, reuse: bool,
                 zero_ptr: tp.Optional[int], zero_count: int, virial: tp.Optional[Tensor],
                 run: tp.Callable[[str, tp.Callable[[], int]], None], refresh_stage: str = "prepare_step"
                 ) -> tp.Tuple[tp.Any, ...]:
        """Enqueue the step's preparation: bucket grid + species-grouped row layout + live AEV column blocks, and the
        zero-fill of the ``zero_count`` floats at ``zero_ptr`` (the force accumulator) and of ``virial`` -- one fused
        entry point -- or, with a Verlet skin and reuse=True, one launch that only refreshes the positions inside the
        grid of an earlier step (stage ``refresh_stage``).  ``run(name, fn)`` launches the stage.  Returns the extra arguments of the AEV entry
        points: in grid mode 3 (one cell per conformer) the same kernels run through the ``_cells`` entry points, which
        take the lattice table the preparation writes (the cells are read from the workspace by the preparation,
        inside a captured graph)."""
        L, c = self.lib, self.consts
        n, n_conf, n_per_conf = ws.n, ws.n_conf, ws.n_per_conf
        st = torch.cuda.current_stream(self.device).cuda_stream
        mode = _grid_mode(n_conf, pbc, conformer_cells)
        prepare, cell_ptr, lat = L.ani_b200_prepare_step, ptr(ws.cell) if pbc else None, ()
        if mode == 3:
            prepare, cell_ptr, lat = L.ani_b200_prepare_step_cells, ptr(ws.cells), (ptr(ws.lattice),)
        if reuse:
            run(refresh_stage, lambda: L.ani_b200_verlet_positions(
                1, ptr(ws.coords), ptr(ws.grid), ptr(ws.sorted_orig), n, self.skin, ptr(ws.spos), ptr(ws.ref_pos),
                ptr(ws.ref_shift), ptr(ws.moved), zero_ptr, zero_count, ptr(ws.aev_blocks), self.nets.ldx, st))
        else:
            run("prepare_step", lambda: prepare(
                ptr(ws.coords), ptr(ws.species_i32), n_conf, n_per_conf, cell_ptr, int(bool(pbc)), mode,
                c.rcr + self.skin, ws.max_bins, ptr(ws.grid), ptr(ws.bin_start), ptr(ws.sorted_orig),
                ptr(ws.orig_to_sorted), ptr(ws.spos), ptr(ws.sbin), ptr(ws.bucket_ranges),
                lo, hi, c.num_species, ws.rows_cap, ptr(ws.row_of), ptr(ws.row_atom), ptr(ws.tile_species),
                ptr(ws.layout_info), len(c.shf_r), len(c.shf_a) * len(c.shf_z), c.out_dim, self.nets.ldx,
                self.nets.col_pad, ptr(ws.aev_blocks), zero_ptr, zero_count,
                ptr(virial) if virial is not None else None, virial.numel() if virial is not None else 0,
                ptr(ws.bucket_species), ptr(ws.scratch), ptr(ws.status), *lat, st))
            if self.skin > 0:
                check(L.ani_b200_verlet_positions(
                    0, ptr(ws.coords), ptr(ws.grid), ptr(ws.sorted_orig), n, self.skin, ptr(ws.spos),
                    ptr(ws.ref_pos), ptr(ws.ref_shift), ptr(ws.moved), None, 0, None, self.nets.ldx, st),
                    "verlet_positions")
        return lat

    def _aev_forward(self, ws: Workspace, lo: int, hi: int, reuse: bool, lat: tp.Tuple[tp.Any, ...],
                     run: tp.Callable[[str, tp.Callable[[], int]], None]) -> None:
        """Enqueue the AEV forward of atoms [lo, hi) into ``ws.x`` (``lat`` as returned by ``_prepare``)."""
        L = self.lib
        aev_forward = L.ani_b200_aev_forward_cells if lat else L.ani_b200_aev_forward
        run("aev_forward", lambda: aev_forward(
            C.byref(self.params), ptr(ws.grid), ptr(ws.bin_start), ptr(ws.spos), ptr(ws.sbin),
            ptr(ws.bucket_ranges), ptr(ws.bucket_species) if not reuse else None,
            ws.aev_blocks.data_ptr() + 4 * (ws.n_blocks + 1), ws.n, lo, hi,
            ptr(ws.row_of), ptr(ws.x), self.nets.ldx, 1, ptr(ws.nbr_cnt), ptr(ws.nbr_list), ws.nbr_cap,
            ptr(ws.status), *lat, torch.cuda.current_stream(self.device).cuda_stream))

    def _launch(self, ws: Workspace, pbc: bool, want_grad: bool, lo: int, hi: int, reuse: bool = False,
                want_virial: bool = False, conformer_cells: bool = False, members: bool = False,
                charges: bool = False) -> None:
        """Enqueue the kernels of one step on the current stream (graph-capturable: no allocation,
        no synchronisation, only this library's launches and two memsets)."""
        if members:
            self._launch_members(ws, pbc, reuse, conformer_cells)
            return
        L = self.lib
        n, n_conf, n_per_conf = ws.n, ws.n_conf, ws.n_per_conf
        st = torch.cuda.current_stream(self.device).cuda_stream
        lat = self._prepare(ws, pbc, conformer_cells, lo, hi, reuse, ws.grad_ptr if want_grad else None,
                            3 * n if want_grad else 0, ws.virial if want_virial else None, self._timed)
        aev_backward = L.ani_b200_aev_backward_cells if lat else L.ani_b200_aev_backward
        # Two small kernels leave the critical path on a side stream (forked and joined with events, so
        # the whole thing still captures into one CUDA graph): the zero-fill of dE/dAEV runs beside the
        # AEV forward / forward GEMMs, the energy reduction beside the backward GEMMs / AEV backward.
        main = torch.cuda.current_stream(self.device)
        side = main if (self.profile or not self.side_stream) else self._side()
        split = side is not main
        zero_first = want_grad and self.nets.num_members > 1
        if split and zero_first:
            self._ev[0].record(main)
            side.wait_event(self._ev[0])
            check(L.ani_b200_zero_live_blocks(C.byref(self.nets.model), ptr(ws.dx), ptr(ws.layout_info),
                                              ptr(ws.aev_blocks), side.cuda_stream), "zero_live_blocks")
            self._ev[1].record(side)
        self._aev_forward(ws, lo, hi, reuse, lat, self._timed)

        def reduce_on(stream_handle):
            return L.ani_b200_reduce_energies(
                C.byref(self.nets.model), ptr(ws.e_member), ws.rows_cap, ptr(ws.row_of), ptr(ws.orig_to_sorted),
                ptr(ws.species_i32), n, lo, hi, n_conf, n_per_conf, ptr(self.sae), ptr(ws.atomic),
                ptr(ws.member_atomic), ws.energies_ptr, stream_handle)

        self.mlp_resident = not split and self._use_resident_mlp(hi - lo, want_grad)
        self.mlp_fused = self.mlp_resident or self._use_dataflow_mlp(hi - lo)
        if self.mlp_resident:
            # the six GEMMs of the step as ONE launch of resident (row tile, member) chains (csrc/mlp_resident.cuh)
            self._timed("mlp_forward_backward", lambda: L.ani_b200_mlp_step_resident(
                C.byref(self.nets.model), ptr(ws.x), ptr(ws.dx), ws.rows_cap, ptr(ws.row_atom),
                ptr(ws.layout_info), ptr(ws.aev_blocks), ptr(ws.act1), ptr(ws.act2), ptr(ws.e_member),
                ptr(ws.status), st))
        elif not split and self.mlp_fused:
            # the six GEMMs of the step as ONE persistent data-flow launch (csrc/gemm_tc.cuh)
            self._timed("mlp_forward_backward", lambda: L.ani_b200_mlp_step(
                C.byref(self.nets.model), ptr(ws.x), ptr(ws.dx), ws.rows_cap, ptr(ws.row_atom),
                ptr(ws.layout_info), ptr(ws.aev_blocks), ptr(ws.act1), ptr(ws.act2), ptr(ws.act3), ptr(ws.e_member),
                int(want_grad), ptr(ws.mlp_sync), ptr(ws.status), st))
        elif not split:
            self._timed("mlp_forward_backward", lambda: L.ani_b200_mlp_forward_backward(
                C.byref(self.nets.model), ptr(ws.x), ptr(ws.dx), ws.rows_cap, ptr(ws.row_atom),
                ptr(ws.layout_info), ptr(ws.aev_blocks), ptr(ws.act1), ptr(ws.act2), ptr(ws.act3), ptr(ws.e_member),
                int(want_grad), ptr(ws.status), st))
        else:
            check(L.ani_b200_mlp_forward(
                C.byref(self.nets.model), ptr(ws.x), ws.rows_cap, ptr(ws.row_atom), ptr(ws.layout_info),
                ptr(ws.aev_blocks), ptr(ws.act1), ptr(ws.act2), ptr(ws.act3), ptr(ws.e_member), int(want_grad),
                ptr(ws.status), st), "mlp_forward")
            self._ev[2].record(main)
            side.wait_event(self._ev[2])
            check(reduce_on(side.cuda_stream), "reduce_energies")
            self._ev[3].record(side)
            if want_grad:
                if zero_first:
                    main.wait_event(self._ev[1])
                check(L.ani_b200_mlp_backward(
                    C.byref(self.nets.model), ptr(ws.dx), ws.rows_cap, ptr(ws.row_atom), ptr(ws.layout_info),
                    ptr(ws.aev_blocks), ptr(ws.act1), ptr(ws.act2), ptr(ws.act3), int(zero_first), ptr(ws.status), st),
                    "mlp_backward")
        # the energy reduction only needs the MLP's forward outputs: beside the AEV backward (a forked branch of the
        # captured graph), not after it
        overlap = want_grad and not split and self.overlap_reduce and not self.profile
        if overlap:
            side2 = self._side()
            self._ev[2].record(main)
            side2.wait_event(self._ev[2])
            check(reduce_on(side2.cuda_stream), "reduce_energies")
            self._ev[3].record(side2)
        if want_grad:
            self._timed("aev_backward", lambda: aev_backward(
                C.byref(self.params), ptr(ws.grid), ptr(ws.spos), ptr(ws.sorted_orig),
                ws.aev_blocks.data_ptr() + 4 * (ws.n_blocks + 1), n, lo, hi,
                ptr(ws.row_of), ptr(ws.dx), self.nets.ldx, ptr(ws.nbr_cnt), ptr(ws.nbr_list), ws.nbr_cap,
                ws.grad_ptr, ptr(ws.status), ws.max_elements, ptr(ws.virial) if want_virial else None, *lat, st))
        if overlap or split:
            main.wait_event(self._ev[3])
        else:
            self._timed("reduce_energies", lambda: reduce_on(st))
        if self.pairs:
            self._pair_potentials(ws, lo, hi, lat, ws.grad_ptr if want_grad else None,
                                  ptr(ws.virial) if want_virial else None, None, self._timed)
        if self.search_pairs:
            self._search_pairs(ws, lo, hi, lat, ws.grad_ptr if want_grad else None,
                               ptr(ws.virial) if want_virial else None, None, self._timed)
        if self.dispersion is not None:
            self._dispersion(ws, lo, hi, lat, ws.grad_ptr if want_grad else None,
                             ptr(ws.virial) if want_virial else None, None, self._timed)
        if charges:
            self._charge_pass(ws, self._timed)
        if ws.reducer is not None:
            # multi-GPU: sum the partial forces / energies of all ranks over NVLink peer memory (one launch,
            # part of the captured graph); without forces only the energies matter but the buffer is small
            def reduce_all() -> int:
                ws.reducer.launch(ws.grad, ws.energies)
                return 0
            self._timed("allreduce", reduce_all)

    def _pair_potentials(self, ws: Workspace, lo: int, hi: int, lat: tp.Tuple[tp.Any, ...], grad_ptr: tp.Optional[int],
                         virial_ptr: tp.Optional[int], grad_members_ptr: tp.Optional[int],
                         run: tp.Callable[[str, tp.Callable[[], int]], None]) -> None:
        """Enqueue the model's pair potentials for atoms [lo, hi): one launch each over the neighbour words the AEV
        forward left in the workspace, adding to the atomic / conformer energies, to every active member's atomic
        energies (the reference adds a pair potential to every member, arch.py:365-378), to the gradient and the
        virial and -- the query-by-committee step -- to every member's gradient.  The kernel adds by plain
        read-modify-write, so it goes on the main stream after the AEV backward and the energy reduction and before
        the statistics / the all-reduce."""
        L = self.lib
        st = torch.cuda.current_stream(self.device).cuda_stream
        active = list(self.nets.active)
        idx = (C.c_int32 * len(active))(*active)
        fn = L.ani_b200_pair_potential_cells if lat else L.ani_b200_pair_potential
        for p in self.pairs:
            run("pair_potential", lambda p=p: fn(
                C.byref(p), ptr(ws.grid), ptr(ws.spos), ptr(ws.sorted_orig), ws.n, lo, hi, ws.n_conf, ws.n_per_conf,
                ptr(ws.nbr_cnt), ptr(ws.nbr_list), ws.nbr_cap, ptr(ws.atomic), ws.energies_ptr, grad_ptr, virial_ptr,
                ptr(ws.member_atomic), grad_members_ptr, idx, len(active), *lat, st))

    def _search_pairs(self, ws: Workspace, lo: int, hi: int, lat: tp.Tuple[tp.Any, ...], grad_ptr: tp.Optional[int],
                      virial_ptr: tp.Optional[int], grad_members_ptr: tp.Optional[int],
                      run: tp.Callable[[str, tp.Callable[[], int]], None]) -> None:
        """Enqueue the LJ / Coulomb pair potentials for atoms [lo, hi): one launch each of
        ani_b200_pair_potential_search (a neighbour search of the potential's own cutoff over the step's bucket grid,
        reach cutoff + ``skin``), with the outputs and the ordering rules of ``_pair_potentials``.  A cell thinner than
        the cutoff + skin raises ANI_STATUS_CELL_TOO_SMALL (``check_status``)."""
        L = self.lib
        st = torch.cuda.current_stream(self.device).cuda_stream
        active = list(self.nets.active)
        idx = (C.c_int32 * len(active))(*active)
        fn = L.ani_b200_pair_potential_search_cells if lat else L.ani_b200_pair_potential_search
        for p in self.search_pairs:
            run("pair_potential_search", lambda p=p: fn(
                C.byref(p), ptr(ws.grid), ptr(ws.bin_start), ptr(ws.spos), ptr(ws.sorted_orig), ws.n, lo, hi,
                ws.n_conf, ws.n_per_conf, self.skin, ptr(ws.atomic), ws.energies_ptr, grad_ptr, virial_ptr,
                ptr(ws.member_atomic), grad_members_ptr, idx, len(active), ptr(ws.status), *lat, st))

    def _dispersion(self, ws: Workspace, lo: int, hi: int, lat: tp.Tuple[tp.Any, ...], grad_ptr: tp.Optional[int],
                    virial_ptr: tp.Optional[int], grad_members_ptr: tp.Optional[int],
                    run: tp.Callable[[str, tp.Callable[[], int]], None]) -> None:
        """Enqueue the D3 term for atoms [lo, hi) (ani_b200_dispersion_d3: its own neighbour search over the step's
        bucket grid, reach cutoff + ``skin``) with the outputs and the ordering rules of ``_pair_potentials``.  A cell
        thinner than the D3 cutoff + skin raises ANI_STATUS_CELL_TOO_SMALL (``check_status``)."""
        L = self.lib
        st = torch.cuda.current_stream(self.device).cuda_stream
        active = list(self.nets.active)
        idx = (C.c_int32 * len(active))(*active)
        fn = L.ani_b200_dispersion_d3_cells if lat else L.ani_b200_dispersion_d3
        params, tables = self.dispersion
        run("dispersion_d3", lambda: fn(
            C.byref(params), ptr(tables), ptr(ws.grid), ptr(ws.bin_start), ptr(ws.spos), ptr(ws.sorted_orig), ws.n, lo,
            hi, ws.n_conf, ws.n_per_conf, self.skin, ptr(ws.d3_cn), ptr(ws.d3_dedcn), ptr(ws.atomic), ws.energies_ptr,
            grad_ptr, virial_ptr, ptr(ws.member_atomic), grad_members_ptr, idx, len(active), ptr(ws.status), *lat, st))

    def set_charges(self, charges: tp.Optional[tp.Tuple[PackedNetworks, ChargeParams]]) -> None:
        """Attach (or replace) the charge networks and the normaliser / dipole parameters (see ``__init__``)."""
        if charges is not None:
            qn, qp = charges
            nets = self.nets
            if qn.num_members != 1:
                raise ValueError("the charge networks must be one member")
            if (qn.in_dim, qn.num_species, qn.ldx, qn.col_pad, qn.variant) != (
                    nets.in_dim, nets.num_species, nets.ldx, nets.col_pad, nets.variant):
                raise ValueError("the charge networks must read the energy networks' AEV operand: same AEV length, "
                                 "elements, internal column order and operand format")
            if len(qp.weights) != nets.num_species or (qp.masses is not None and len(qp.masses) != nets.num_species):
                raise ValueError("one normaliser weight (and mass) per element is required")
            if qp.frame not in (0, 1, 2) or (qp.frame == 0 and qp.masses is None):
                raise ValueError("the centre-of-mass dipole frame needs one mass per element")
        self.charges = charges

    def charge_buffers(self, ws: Workspace) -> None:
        """Allocate the charge networks' activations and raw outputs (once per workspace, before any capture)."""
        if ws.q_raw is None:
            qn = self.charges[0]
            ws.q_act = tuple(operand_buffer(ws.rows_cap, w, self.device, self.variant) for w in qn.act_cols)
            ws.q_raw = torch.zeros(1, ws.rows_cap, dtype=torch.float32, device=self.device)

    def _charge_launches(self, ws: Workspace) -> int:
        """Kernels a step with charges adds: the forward-only charge network pass and ani_b200_charges."""
        if self.charge_mlp == "step":
            return self.lib.ani_b200_mlp_step_windows(C.byref(self.charges[0].model), ws.rows_cap) + 1
        return 3 + 1

    def _charge_pass(self, ws: Workspace, run: tp.Callable[[str, tp.Callable[[], int]], None]) -> None:
        """Enqueue the charge networks (forward only, one member) on the step's tiled AEVs ``ws.x`` and live column
        blocks, then ani_b200_charges: normalised charges in input order and one dipole per conformer.  It goes after
        every other kernel of the step: none of them writes ``ws.x`` after the AEV forward (the MLP reads it, the AEV
        backward, the pair and D3 terms read ``dx`` / the neighbour words), so the energy step's own launches and
        their order are those of a step without charges."""
        if self.charge_mlp not in ("chained", "step"):
            raise ValueError(f"ANI_B200_CHARGE_MLP={self.charge_mlp!r}: expected 'chained' or 'step'")
        L = self.lib
        qn, qp = self.charges
        st = torch.cuda.current_stream(self.device).cuda_stream
        a1, a2, a3 = ws.q_act
        if self.charge_mlp == "step":
            run("charge_forward", lambda: L.ani_b200_mlp_step(
                C.byref(qn.model), ptr(ws.x), None, ws.rows_cap, ptr(ws.row_atom), ptr(ws.layout_info),
                ptr(ws.aev_blocks), ptr(a1), ptr(a2), ptr(a3), ptr(ws.q_raw), 0, ptr(ws.mlp_sync), ptr(ws.status), st))
        else:
            run("charge_forward", lambda: L.ani_b200_mlp_forward(
                C.byref(qn.model), ptr(ws.x), ws.rows_cap, ptr(ws.row_atom), ptr(ws.layout_info), ptr(ws.aev_blocks),
                ptr(a1), ptr(a2), ptr(a3), ptr(ws.q_raw), 0, ptr(ws.status), st))
        w, m = qp.arrays()
        run("charges", lambda: L.ani_b200_charges(
            ptr(ws.q_raw), ptr(ws.row_of), ptr(ws.orig_to_sorted), ptr(ws.species_i32), ptr(ws.coords), ws.n_conf,
            ws.n_per_conf, w, qn.num_species, int(qp.scale_by_q2), int(qp.normalize), 0.0, m, qp.frame,
            ptr(ws.charges), ptr(ws.dipoles), st))

    def charges_result(self, ws: Workspace) -> ChargesResult:
        """Views of the charges and dipoles of the last ``run(..., charges=True)`` on ``ws``."""
        assert ws.q_raw is not None, "no step with charges has run on this workspace"
        return ChargesResult(ws.charges.view(ws.n_conf, ws.n_per_conf), ws.dipoles)

    def raw_charges(self, ws: Workspace) -> Tensor:
        """(C, A) float32 raw charges (the charge networks' outputs before the normaliser) of the last step with
        charges, in input order, 0 for padding (a gather on the stream; for tests and diagnostics)."""
        assert ws.q_raw is not None, "no step with charges has run on this workspace"
        sp = ws.species_i32
        rows = ws.row_of.long()[ws.orig_to_sorted.long().clamp(min=0)]
        q = torch.where(sp >= 0, ws.q_raw[0][rows.clamp(min=0)], torch.zeros_like(ws.q_raw[0][:1]))
        return q.view(ws.n_conf, ws.n_per_conf)

    def members_buffers(self, ws: Workspace) -> None:
        """Allocate the per-member slabs and gradients of the query-by-committee step (once per workspace, before any
        capture of the step)."""
        M = self.nets.num_members
        if ws.dx_members is None:
            ws.dx_members = torch.zeros(M, ws.rows_cap, self.nets.ldx, dtype=torch.float32, device=self.device)
        if ws.grad_members is None:
            ws.grad_members = torch.zeros(M, ws.n, 3, dtype=torch.float32, device=self.device)

    def _launch_members(self, ws: Workspace, pbc: bool, reuse: bool, conformer_cells: bool) -> None:
        """The query-by-committee step (graph-capturable like _launch): preparation (or the Verlet refresh) that zeroes
        the members' gradients, AEV forward, ONE MLP launch whose layer-1 backward writes a dE_m/dAEV slab per active
        member with unit weight (the resident chains of ani_b200_mlp_step_resident_members where the ordinary step
        would run ani_b200_mlp_step_resident, else ani_b200_mlp_step with want_backward=2), ONE AEV backward over every
        active member's slab
        (ani_b200_aev_backward_members), the energy reduction (ensemble mean, per-member atomic energies) and the
        statistics kernel, which also writes the ensemble-mean gradient into ``ws.grad``."""
        L = self.lib
        n, n_conf, n_per_conf = ws.n, ws.n_conf, ws.n_per_conf
        st = torch.cuda.current_stream(self.device).cuda_stream
        nets = self.nets
        active = list(nets.active)
        Ma = len(active)
        idx = (C.c_int32 * Ma)(*active)
        gm = ptr(ws.grad_members)

        def run(name: str, fn: tp.Callable[[], int]) -> None:   # no profile events in this step
            check(fn(), name)
        lat = self._prepare(ws, pbc, conformer_cells, 0, n, reuse, gm, 3 * n * Ma, None, run, "verlet_positions")
        self._aev_forward(ws, 0, n, reuse, lat, run)
        backward = L.ani_b200_aev_backward_members_cells if lat else L.ani_b200_aev_backward_members
        mask_ptr = ws.aev_blocks.data_ptr() + 4 * (ws.n_blocks + 1)
        unit = _lib.MLPModel.from_buffer_copy(nets.model)     # every active member with weight 1 (not 1 / M)
        for m in range(_lib.ANI_MAX_MEMBERS):
            unit.member_scale[m] = 1.0 if m in active else 0.0
        self.mlp_resident = self._use_resident_mlp(n, True)
        if self.mlp_resident:
            check(L.ani_b200_mlp_step_resident_members(
                C.byref(unit), ptr(ws.x), ptr(ws.dx_members), ws.rows_cap * nets.ldx, ws.rows_cap, ptr(ws.row_atom),
                ptr(ws.layout_info), ptr(ws.aev_blocks), ptr(ws.act1), ptr(ws.act2), ptr(ws.e_member), ptr(ws.status),
                st), "mlp_step_resident_members")
        else:
            check(L.ani_b200_mlp_step(
                C.byref(unit), ptr(ws.x), ptr(ws.dx_members), ws.rows_cap, ptr(ws.row_atom), ptr(ws.layout_info),
                ptr(ws.aev_blocks), ptr(ws.act1), ptr(ws.act2), ptr(ws.act3), ptr(ws.e_member), 2, ptr(ws.mlp_sync),
                ptr(ws.status), st), "mlp_step")
        check(backward(
            C.byref(self.params), ptr(ws.grid), ptr(ws.spos), ptr(ws.sorted_orig), mask_ptr, n, 0, n,
            ptr(ws.row_of), ptr(ws.dx_members), nets.ldx, ws.rows_cap * nets.ldx, idx, Ma, ptr(ws.nbr_cnt),
            ptr(ws.nbr_list), ws.nbr_cap, gm, ptr(ws.status), ws.max_elements, *lat, st), "aev_backward_members")
        check(L.ani_b200_reduce_energies(
            C.byref(nets.model), ptr(ws.e_member), ws.rows_cap, ptr(ws.row_of), ptr(ws.orig_to_sorted),
            ptr(ws.species_i32), n, 0, n, n_conf, n_per_conf, ptr(self.sae), ptr(ws.atomic), ptr(ws.member_atomic),
            ws.energies_ptr, st), "reduce_energies")
        if self.pairs:   # before the statistics: they read the members' atomic energies and gradients
            self._pair_potentials(ws, 0, n, lat, None, None, gm, run)
        if self.search_pairs:
            self._search_pairs(ws, 0, n, lat, None, None, gm, run)
        if self.dispersion is not None:
            self._dispersion(ws, 0, n, lat, None, None, gm, run)
        check(L.ani_b200_ensemble_qbc(
            gm, idx, Ma, ptr(ws.member_atomic), ptr(ws.species_i32), ptr(self.sae), n_conf, n_per_conf,
            ptr(ws.grad), ptr(ws.atom_stats), ptr(ws.member_energies), ptr(ws.qbc), st), "ensemble_qbc")

    def members_result(self, ws: Workspace) -> MembersResult:
        """Views of the query-by-committee outputs of the last ``run(..., members=True)`` on ``ws``."""
        Ma, C_, A = len(self.nets.active), ws.n_conf, ws.n_per_conf
        assert ws.grad_members is not None, "no query-by-committee step has run on this workspace"
        st = ws.atom_stats.view(3, C_, A)
        return MembersResult(ws.member_energies[:Ma], ws.grad_members[:Ma].view(Ma, C_, A, 3), ws.qbc, st[0], st[1],
                             st[2])

    def step_members(self, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None, pbc: bool = False
                     ) -> tp.Tuple[Tensor, Tensor]:
        """Energies (M_active, C) float64 and dE_m/dcoords (M_active, C, A, 3) float32 of every ACTIVE ensemble member
        (arch.py:403-436 differentiates every member by autograd): the query-by-committee step,
        ``run(..., members=True)`` -- one MLP launch writes a dE_m/dAEV slab per member and ONE AEV backward contracts
        all of them -- captured into a CUDA graph like the ordinary step."""
        with torch.cuda.device(self.device):
            ws, per_conf = self._stage_inputs(species, coords, cell, pbc)
        self.run(ws, bool(pbc), True, members=True, conformer_cells=per_conf)
        r = self.members_result(ws)
        return r.energies.clone(), r.grad.clone()

    # -- analytic Hessians ------------------------------------------------------------------------
    def hessian(self, ws: Workspace, row_budget: int = HESSIAN_ROW_BUDGET) -> Tensor:
        """(C, 3A, 3A) float32 Hessian d^2E/dx^2 of the energies of the last ``run(ws, pbc=False, want_grad=True)`` on
        ``ws`` (an open single molecule or conformer batch, unsharded), in input atom order, accumulated in float64;
        padding atoms get zero rows and columns, conformers are independent blocks.  It reads what that step left in the
        workspace (neighbour words, AEVs, dE/dAEV rows) and runs as eager launches of csrc/hessian.cu, per chunk of
        central atoms whose Jacobian rows (3 per neighbour) fit ``row_budget``: AEV Jacobian rows, the tangent network
        pass of every active member, the geometric and xTB / ZBL terms, and the assembly.  Synchronises once to plan the
        chunks."""
        last = getattr(ws, "last_run", None)
        if last is None:
            raise ValueError("Engine.hessian needs a step with gradients on this workspace first: "
                             "run(ws, pbc=False, want_grad=True)")
        periodic, have_dx, sharded = last
        if periodic:
            raise ValueError("Hessians of periodic systems are not supported (open molecules and conformer batches "
                             "only)")
        if sharded:
            raise ValueError("Hessians are computed on one unsharded engine: every atom's neighbour words and dE/dAEV "
                             "row are needed")
        if not have_dx:
            raise ValueError("Engine.hessian needs the dE/dAEV rows of an ordinary step with gradients "
                             "(run(ws, pbc=False, want_grad=True))")
        if self.dispersion is not None:
            raise NotImplementedError("Hessians of models with D3 dispersion are not supported")
        if self.search_pairs:
            raise NotImplementedError("Hessians of models with Lennard-Jones or Coulomb pair potentials (kinds 2-6) "
                                      "are not supported; only the xTB and ZBL repulsion terms have second "
                                      "derivatives")
        L, nets = self.lib, self.nets
        dev = self.device
        n_conf, A = ws.n_conf, ws.n_per_conf
        with torch.cuda.device(dev):
            st = torch.cuda.current_stream(dev).cuda_stream
            n_real = int(self.grid_info(ws).n_real)
            cnt = ws.nbr_cnt[:n_real].clamp(max=ws.nbr_cap).cpu().numpy().astype(np.int64)
            species = ws.spos[:n_real, 3].contiguous().view(torch.int32).cpu().numpy()
            hess = torch.zeros(n_conf, 3 * A, 3 * A, dtype=torch.float64, device=dev)
            hmax = L.ani_b200_hessian_hidden_max(C.byref(nets.model))
            pairs = [torch.frombuffer(bytearray(bytes(p)), dtype=torch.uint8).to(dev) for p in self.pairs]
            for chunk in _hessian_chunks(cnt, species, int(row_budget)):
                self._hessian_chunk(ws, chunk, hmax, pairs, hess, st)
        self.hessian_count += 1
        return hess.to(torch.float32)

    def hessian_chunk_args(self, plan: "_HessianPlan") -> tp.Tuple[_lib.HessianChunk, tp.List[Tensor]]:
        """The ani_hessian_chunk of ``plan`` and the device arrays it points into (keep them alive while it is used)."""
        dev = self.device
        i32 = torch.from_numpy(np.concatenate([plan.atom, plan.row_off, plan.row_slot, plan.tile_species])).to(dev)
        b_off = torch.from_numpy(plan.block_off).to(dev)
        ns, rows = len(plan.atom), plan.rows
        ch = _lib.HessianChunk()
        ch.atom, ch.row_off = i32.data_ptr(), i32.data_ptr() + 4 * ns
        ch.row_slot, ch.tile_species = i32.data_ptr() + 8 * ns, i32.data_ptr() + 4 * (2 * ns + rows)
        ch.block_off = b_off.data_ptr()
        ch.n_slots, ch.rows, ch.max_count = ns, rows, plan.max_count
        return ch, [i32, b_off]

    def _hessian_chunk(self, ws: Workspace, plan: "_HessianPlan", hmax: int, pairs: tp.List[Tensor], hess: Tensor,
                       st: int) -> None:
        """Enqueue the four stages of one chunk of central atoms (see ``hessian``)."""
        L, nets, dev = self.lib, self.nets, self.device
        ch, _keep = self.hessian_chunk_args(plan)
        ns, rows = len(plan.atom), plan.rows
        jac = torch.empty(rows, nets.ldx, dtype=torch.float32, device=dev)
        scratch = torch.empty(4 * rows * hmax + ns * 5 * hmax, dtype=torch.float32, device=dev)
        blocks = torch.zeros(plan.block_floats, dtype=torch.float32, device=dev)
        cap = ws.nbr_cap
        self._timed("hessian_jacobian", lambda: L.ani_b200_hessian_jacobian(
            C.byref(self.params), ptr(ws.spos), ptr(ws.nbr_cnt), ptr(ws.nbr_list), cap, C.byref(ch), ptr(jac),
            nets.ldx, st))
        self._timed("hessian_network", lambda: L.ani_b200_hessian_network(
            C.byref(nets.model), C.byref(nets.plain_weights), ptr(ws.x), ptr(ws.row_of), ptr(ws.spos), ptr(ws.nbr_cnt),
            cap, C.byref(ch), ptr(jac), ptr(scratch), ptr(blocks), st))
        self._timed("hessian_geometric", lambda: L.ani_b200_hessian_geometric(
            C.byref(self.params), ptr(ws.spos), ptr(ws.nbr_cnt), ptr(ws.nbr_list), cap, ptr(ws.row_of), ptr(ws.dx),
            nets.ldx, None, C.byref(ch), ptr(blocks), st))
        for p in pairs:
            self._timed("hessian_geometric", lambda p=p: L.ani_b200_hessian_geometric(
                C.byref(self.params), ptr(ws.spos), ptr(ws.nbr_cnt), ptr(ws.nbr_list), cap, None, None, 0, ptr(p),
                C.byref(ch), ptr(blocks), st))
        self._timed("hessian_assemble", lambda: L.ani_b200_hessian_assemble(
            ptr(ws.nbr_cnt), ptr(ws.nbr_list), cap, ptr(ws.sorted_orig), C.byref(ch), ptr(blocks), ws.n_per_conf,
            ptr(hess), st))

    def _use_dataflow_mlp(self, owned: int) -> bool:
        """One data-flow launch (True) or six chained launches (False) for `owned` atoms; see __init__."""
        if self.mlp_mode in ("0", "1"):
            return self.mlp_mode == "1"
        units = (-(-owned // TILE) + 1) * self.nets.num_members     # per layer: row tiles x members (>= 1 column tile)
        return units >= self._num_sms

    def _use_resident_mlp(self, owned: int, want_grad: bool) -> bool:
        """One launch of resident chains (ani_b200_mlp_step_resident) where "auto" would pick the data-flow launch
        for a step with gradients, and the build and the model have the kernel; see __init__."""
        return self.mlp_mode == "auto" and want_grad and self._resident_ok and self._use_dataflow_mlp(owned)

    def note_composition(self, ws: Workspace) -> None:
        """Before a graph capture (the shape has already run eagerly): read the element mask of the last
        step once and let the AEV backward size its shared-memory gradient table for that many elements
        (more elements at replay time still give the right answer, from global memory)."""
        mask = int(ws.aev_blocks[ws.n_blocks + 1].item())
        ws.max_elements = bin(mask).count("1")

    def _side(self) -> "torch.cuda.Stream":
        if self._side_stream is None:
            self._side_stream = torch.cuda.Stream(self.device)
            self._ev = [torch.cuda.Event() for _ in range(4)]
        return self._side_stream

    # -- status ----------------------------------------------------------------------------
    def check_status(self, ws: tp.Optional[Workspace] = None) -> None:
        """Raise for device-side conditions (one D2H read; call when results are consumed)."""
        for w in ([ws] if ws is not None else list(self._ws.values())):
            code = int(w.status.item())
            if code == 0:
                continue
            w.status.zero_()
            if code & _lib.STATUS_CELL_TOO_SMALL:
                raise RuntimeError("Cell is too small to perform pbc calculations")  # neighbors.py:402-403
            if code & _lib.STATUS_NBR_OVERFLOW:
                raise RuntimeError(f"an atom has more than nbr_cap={w.nbr_cap} neighbours within Rcr; "
                                   "construct the engine with a larger nbr_cap (<= 256)")
            if code & _lib.STATUS_ANG_OVERFLOW:
                raise RuntimeError(f"an atom has more than {_lib.ANI_MAX_ANG} neighbours within Rca")
            if code & _lib.STATUS_PAIR_OVERFLOW:
                raise RuntimeError("half neighbour list capacity exceeded")
            if code & _lib.STATUS_INTERNAL:
                raise RuntimeError("a device-side barrier of libani_b200 timed out (internal error)")
            if code & _lib.STATUS_OPERAND_RANGE:
                raise _lib.OperandRangeError(
                    "an AEV, activation or gradient left the range of the half-precision GEMM operand pieces "
                    "(inf/NaN input, or |value| > 1023.5 / |gradient| > 65504 / 4096); the 3 x bfloat16 build of the library "
                    "(variant 'bf16x3') has no such limit -- models.ANI switches to it automatically")

    def grid_info(self, ws: Workspace) -> Grid:
        g = Grid()
        raw = ws.grid.cpu().numpy().tobytes()
        C.memmove(C.byref(g), raw, C.sizeof(Grid))
        return g
