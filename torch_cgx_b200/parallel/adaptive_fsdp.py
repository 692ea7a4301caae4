"""Adaptive per-parameter bit widths for the FSDP2 reduce-scatter and all-gather.

``AdaptiveFSDPState`` keeps each kind's *average* width (``reduce_scatter_bits``,
``all_gather_bits``) but moves bits to the parameters where quantization hurts most. It is the
FSDP2 counterpart of :class:`~torch_cgx_b200.AdaptiveCGXState`::

    model = fully_shard(model)
    state = cgx.AdaptiveFSDPState(reduce_scatter_bits=4, all_gather_bits=6, period=1000)
    comms = cgx.set_cgx_adaptive(model, state)   # after fully_shard, before the first forward

Rounds. Every root forward is one step. A round opens at the root pre-forward of every step that is
a multiple of ``period``. While it is open, each comm estimates, on its next compressed call, the
per-parameter error of what that call quantizes (``ops.quantization_error``, one launch, enqueued on
the stream the collective runs on, before it):

* the all-gather: its shard input, rounded to nearest (the all-gather is never stochastic);
* the reduce-scatter: its whole input in sharded mode (``chunks = world``, ``skip_chunk = rank``:
  rank r sends every chunk but its own), prescaled by 1/world when averaging, with the state's
  rounding mode.

A round is complete once every comm that has made a compressed call holds its estimate; with
gradient accumulation the reduce-scatter's comes from the next sync microbatch. FSDP2 is SPMD, so
every rank completes a round at the same step.

Decision. At the first root pre-forward after a round completes, the estimates are summed over the
group in one float64 ``all_reduce``, group rank 0 picks the widths per kind (``ops.allocate_bits``:
least total error within the wire bytes of the kind's uniform width) and broadcasts them, and every
rank rewrites its comms' shard tables with the broadcast widths. Only broadcast widths are ever
applied, and only at a root pre-forward: every rank uses the same table in every collective, and a
module's forward gather and backward re-gather in one step use the same table.

Limits:

* Estimate and decision steps cannot run inside CUDA graph capture (they raise); calls outside a
  round stay capturable.
* All comms of one state must see one process group. HSDP (a replicate mesh dimension) is not
  supported.
* Over several nodes the reduce-scatter runs in two stages and a remote value is quantized up to
  twice (DESIGN §2.9b); the estimate models the single-stage reduce-scatter, so it is an
  approximation there.
* With a target width equal to the largest candidate, the budget admits only the uniform table.
* An all-gather table with a width outside {2, 4, 8} does not use the NVLink multicast publish.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from ..ops.bit_allocation import layer_wire_bytes
from ..ops.quantization import quantization_error
from .adaptive import _capturing, _sum_allocate_broadcast
from .fsdp import CGXAllGather, CGXReduceScatter, fsdp_shard_table

KINDS = ("reduce_scatter", "all_gather")


class AdaptiveFSDPState:
    """Adaptive widths of the FSDP2 comms (see the module docstring).

    ``reduce_scatter_bits`` / ``all_gather_bits`` are each kind's target width, the average the
    budget is derived from; None leaves that kind's comm alone. After a decision ``assignment`` maps
    ``(kind, parameter name)`` to its width and ``last_errors[kind]`` holds the group-summed error
    table of the kind's estimated rows (float64 ``[rows, len(candidate_bits)]``, rows in
    ``rows(kind)`` order restricted to the comms that estimated)."""

    def __init__(self, reduce_scatter_bits: Optional[int] = 4, all_gather_bits: Optional[int] = 6,
                 bucket_size: int = 512, candidate_bits: Sequence[int] = (2, 3, 4, 5, 6, 7, 8), period: int = 1000,
                 stochastic: bool = False):
        self.targets = {"reduce_scatter": reduce_scatter_bits, "all_gather": all_gather_bits}
        for kind, bits in self.targets.items():
            if isinstance(bits, str):
                raise ValueError(f"{kind}_bits must be a max-min width in 1..8 or None: adaptive widths do not "
                                 f"take FP8 formats, got {bits!r}")
            if bits is not None and not 1 <= int(bits) <= 8:
                raise ValueError(f"{kind}_bits must be a width in 1..8 or None, got {bits}")
        self.targets = {k: None if b is None else int(b) for k, b in self.targets.items()}
        if all(b is None for b in self.targets.values()):
            raise ValueError("AdaptiveFSDPState: reduce_scatter_bits and all_gather_bits are both None")
        self.candidate_bits = tuple(int(b) for b in candidate_bits)
        if not self.candidate_bits or any(b < 1 or b > 8 for b in self.candidate_bits):
            raise ValueError(f"candidate_bits must be widths in 1..8, got {candidate_bits}")
        if bucket_size < 1:
            raise ValueError(f"bucket_size must be >= 1, got {bucket_size}")
        if period < 1:
            raise ValueError(f"period must be >= 1, got {period}")
        self.bucket_size = int(bucket_size)
        self.period = int(period)
        self.stochastic = bool(stochastic)
        self.step = 0
        self.assignment: Dict[Tuple[str, str], int] = {}
        self.last_errors: Dict[str, torch.Tensor] = {}
        self._comms: List = []  # installed comms, in registration order
        self._rows: Dict[int, List[Tuple[int, str]]] = {}  # id(comm) -> (table index, parameter name)
        self._kind: Dict[int, str] = {}
        self._called: set = set()  # ids of comms that made a compressed call
        self._tables: Dict[int, Tuple[torch.Tensor, Optional[torch.cuda.Event]]] = {}
        self._round_open = False
        self._group: Optional[dist.ProcessGroup] = None
        self._loaded: Dict[Tuple[str, str], int] = {}

    # ---- installation ------------------------------------------------------------------------
    def register(self, comm, kind: str, names: Sequence[str]) -> None:
        """Adapt ``comm`` (a :class:`CGXReduceScatter` or :class:`CGXAllGather` with a shard table)
        as ``kind``; ``names[i]`` names table entry i. Entries with bits <= 8 are adapted."""
        if kind not in KINDS:
            raise ValueError(f"unknown kind {kind!r}, expected one of {KINDS}")
        if comm.layers is None or len(names) != len(comm.layers):
            raise ValueError("AdaptiveFSDPState.register: the comm needs a shard table with one name per entry")
        rows = [(i, str(n)) for i, (n, l) in enumerate(zip(names, comm.layers)) if l[2] <= 8]
        comm.adaptive = self
        self._comms.append(comm)
        self._rows[id(comm)] = rows
        self._kind[id(comm)] = kind
        for i, name in rows:
            self.assignment[(kind, name)] = comm.layers[i][2]
        if self._loaded:
            self._apply_loaded(strict=False)

    def rows(self, kind: str) -> List[str]:
        """Names of the adapted parameters of ``kind``, in decision order."""
        return [n for c in self._comms if self._kind[id(c)] == kind for _, n in self._rows[id(c)]]

    # ---- checkpoint -------------------------------------------------------------------------
    def state_dict(self) -> Dict:
        sd: Dict[str, Dict[str, int]] = {k: {} for k in KINDS}
        for (kind, name), bits in self.assignment.items():
            sd[kind][name] = bits
        return {"assignment": sd, "step": self.step}

    def load_state_dict(self, sd: Dict) -> None:
        """Restore ``assignment`` and ``step``. The widths apply to the installed comms at once, or
        to the comms installed later. Unknown kinds or names and widths outside 1..8 raise."""
        loaded = {}
        for kind, widths in dict(sd.get("assignment", {})).items():
            if kind not in KINDS:
                raise ValueError(f"AdaptiveFSDPState.load_state_dict: unknown kind {kind!r}")
            for name, bits in dict(widths).items():
                if not 1 <= int(bits) <= 8:
                    raise ValueError(f"AdaptiveFSDPState.load_state_dict: width {bits} of {kind} {name!r} "
                                     "is outside 1..8")
                loaded[(kind, str(name))] = int(bits)
        self._loaded = loaded
        self.step = int(sd.get("step", self.step))
        if self._comms:
            self._apply_loaded(strict=True)

    def _apply_loaded(self, strict: bool) -> None:
        known = set()
        for c in self._comms:
            kind = self._kind[id(c)]
            for i, name in self._rows[id(c)]:
                known.add((kind, name))
                bits = self._loaded.get((kind, name))
                if bits is not None:
                    self._set_width(c, i, kind, name, bits)
        unknown = sorted(k for k in self._loaded if k not in known)
        if strict and unknown:
            raise ValueError(f"AdaptiveFSDPState.load_state_dict: unknown parameters {unknown[:4]}")

    def _set_width(self, comm, i: int, kind: str, name: str, bits: int) -> None:
        off, n, _, bucket = comm.layers[i]
        comm.layers[i] = (off, n, int(bits), bucket)
        self.assignment[(kind, name)] = int(bits)

    # ---- entry points of the comms and of the root pre-forward --------------------------------
    def maybe_estimate(self, comm, x: torch.Tensor, group: dist.ProcessGroup, average: bool) -> None:
        """Called by an adapted comm before its compressed collective on ``x`` (the all-gather's
        shard input, or the reduce-scatter's whole input). Enqueues the estimate on the current
        stream if a round is open and ``comm`` has none yet."""
        kind = self._kind[id(comm)]
        world = group.size()
        if kind == "reduce_scatter" and world == 1:
            return  # nothing is quantized
        if self._group is None:
            self._group = group
        elif group is not self._group:
            raise RuntimeError("AdaptiveFSDPState: all comms of one state must use one process group "
                               "(HSDP is not supported)")
        self._called.add(id(comm))
        if not self._round_open or id(comm) in self._tables or not self._rows[id(comm)]:
            return
        if _capturing():
            raise RuntimeError("AdaptiveFSDPState: an estimate step cannot run during CUDA graph capture")
        layers = [comm.layers[i] for i, _ in self._rows[id(comm)]]
        if kind == "all_gather":
            t = quantization_error(x, layers, self.candidate_bits)
        else:
            t = quantization_error(x, layers, self.candidate_bits, stochastic=self.stochastic,
                                   prescale=1.0 / world if average else 1.0, chunks=world,
                                   skip_chunk=group.rank())
        ev = None
        if t.is_cuda:
            ev = torch.cuda.Event()
            ev.record()
        self._tables[id(comm)] = (t, ev)

    def pre_forward(self) -> None:
        """The root pre-forward: decide if a round completed, open a round every ``period`` steps."""
        if self._round_open and self._round_complete():
            self._decide()
            self._round_open = False
        if not self._round_open and self.step % self.period == 0:
            self._round_open = True
        self.step += 1

    def _round_complete(self) -> bool:
        return bool(self._tables) and all(i in self._tables for i in self._called if self._rows[i])

    def _decide(self) -> None:
        if _capturing():
            raise RuntimeError("AdaptiveFSDPState: a decision step cannot run during CUDA graph capture")
        stream = torch.cuda.current_stream() if torch.cuda.is_available() else None
        tables, parts, order = [], [], []
        for kind in KINDS:
            comms = [c for c in self._comms if self._kind[id(c)] == kind and id(c) in self._tables]
            if not comms:
                continue
            numels, current, rows = [], [], []
            for c in comms:
                t, ev = self._tables[id(c)]
                if ev is not None:
                    stream.wait_event(ev)
                    t.record_stream(stream)
                tables.append(t)
                for i, name in self._rows[id(c)]:
                    numels.append(c.layers[i][1])
                    current.append(c.layers[i][2])
                    rows.append((c, i, name))
            target = self.targets[kind]
            budget = sum(layer_wire_bytes(n, target, self.bucket_size) for n in numels)
            parts.append((numels, [self.bucket_size] * len(numels), budget, current, target))
            order.append((kind, rows))
        device = tables[0].device
        self._tables = {}
        table, choice = _sum_allocate_broadcast(tables, parts, self.candidate_bits, self._group, device)
        r = 0
        for kind, rows in order:
            for (c, i, name), bits in zip(rows, choice[r:r + len(rows)]):
                self._set_width(c, i, kind, name, bits)
            self.last_errors[kind] = table[r:r + len(rows)]
            r += len(rows)


def set_cgx_adaptive(model: torch.nn.Module, state: AdaptiveFSDPState) -> List:
    """Install an adapted :class:`CGXReduceScatter` and :class:`CGXAllGather` on every
    ``FSDPModule`` of ``model`` that has a parameter group, each with that module's shard table
    (:func:`fsdp_shard_table`) at the kind's target width, and register the state's step counter as
    a forward pre-hook on ``model``, the FSDP root, ahead of FSDP's own. A kind whose target is None
    is left alone. Returns the comms. Call it after ``fully_shard`` and before the first forward."""
    from torch.distributed.fsdp import FSDPModule

    if not isinstance(model, FSDPModule) or model._get_fsdp_state()._is_root is False:
        raise ValueError("set_cgx_adaptive: model must be the FSDP root (fully_shard(model) after its sub-modules)")
    if state._comms:
        raise ValueError("set_cgx_adaptive: the state is installed already")
    names = {id(p): n for n, p in model.named_parameters()}
    comms = []
    for mname, m in model.named_modules():
        if not isinstance(m, FSDPModule):
            continue
        group = m._get_fsdp_state()._fsdp_param_group
        if group is None:  # a module without parameters of its own
            continue
        if getattr(group.mesh_info, "replicate_mesh_dim", None) is not None:
            raise ValueError("set_cgx_adaptive: HSDP (FSDP2 with a replicate mesh dimension) is not supported")
        params = group.fsdp_params
        sizes = [(p._orig_size, p.padded_sharded_param_size.numel()) for p in params]
        fqns = [names[id(p.sharded_param)] for p in params if p.padded_sharded_param_size.numel() > 0]
        label = mname or type(m).__name__
        for kind in KINDS:
            bits = state.targets[kind]
            if bits is None:
                continue
            table = fsdp_shard_table(sizes, bits, state.bucket_size)
            if kind == "reduce_scatter":
                comm = CGXReduceScatter(bits, state.bucket_size, state.stochastic, table, label)
                m.set_custom_reduce_scatter(comm)
            else:
                comm = CGXAllGather(bits, state.bucket_size, table, label)
                m.set_custom_all_gather(comm)
            state.register(comm, kind, fqns)
            comms.append(comm)
    if state._loaded:
        state._apply_loaded(strict=True)
    model.register_forward_pre_hook(lambda module, args: state.pre_forward(), prepend=True)
    return comms
