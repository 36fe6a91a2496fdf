"""Derived bf16 GEMM operands of the fp32 master parameters.

The reference keeps OIHW fp32 ``nn.Parameter``s (checkpoints are plain ``state_dict()``s, classification/resnet/train.py:130),
so the packed [O][taps*I] / [I][taps*O] bf16 copies the tensor cores read are caches, rebuilt whenever a parameter's
version counter or storage changes (optimizer step, ``load_state_dict``) or when ``bump()`` is called by code that updates
parameters behind autograd's back (the fused optimizer kernel).  A model registers all its weights once (``ModelPack``) so
that one multi-tensor launch repacks everything; single tensors fall back to ``ops.pack_weight``.
"""
import weakref

import torch

from .. import ops


class ModelPack:
    """All packed operands of one model, refreshed by ONE kernel launch (b200_pack_weights_multi)."""

    def __init__(self, specs):
        # specs: list of (param, mode, ld, rows_out[, (O, I, taps) override for weights consumed as a flat [O][K] matrix
        #                 [, oscale parameter: fp32 [O] multiplier folded into the packed copy
        #                 [, (name, row, col, rows_total): write into the shared operand ``name`` at (row, col)]]])
        # A shared operand is a zero-initialised [rows_total][ld] matrix that several entries fill (the RepVGG stem's
        # [3x3 | 1x1] operand, read through ``shared(name)``).  An entry at a column offset also writes its zero padding of
        # columns [I*taps, ld) there, which runs into the first ``col`` columns of the next row: those cells must be zero
        # cells no other entry writes, and one spare row takes the last row's overrun.
        self.specs = specs
        self.outputs = {}
        self._shared = {}
        self._ptrs = None
        self.stamp = None
        dev = specs[0][0].device
        rows = []
        first = 0
        for spec in specs:
            p, mode, ld, rows_out = spec[:4]
            if len(spec) > 4 and spec[4] is not None:
                O, I, taps = spec[4]
            else:
                O, I = p.shape[0], p.shape[1]
                taps = p.numel() // (O * I)
            into = spec[6] if len(spec) > 6 else None
            if into is None:
                dst = torch.empty(rows_out, ld, dtype=torch.bfloat16, device=dev)
                self.outputs[(id(p), mode)] = dst
                ptr = dst.data_ptr()
            else:
                name, row, col, rows_total = into
                buf = self._shared.get(name)
                if buf is None:
                    buf = torch.zeros(rows_total + 1, ld, dtype=torch.bfloat16, device=dev)
                    self._shared[name] = buf
                if buf.shape[1] != ld or row + rows_out > rows_total or col + I * taps > ld:
                    raise ValueError(f"ModelPack: entry at ({row}, {col}) of {rows_out} x {I * taps} does not fit the shared "
                                     f"operand {name!r} [{rows_total}][{buf.shape[1]}]")
                ptr = buf.data_ptr() + (row * ld + col) * buf.element_size()
            nblk = max(1, min(64, (rows_out * ld + 256 * 16 - 1) // (256 * 16)))
            rows.append([0, ptr, O, I, taps, mode, ld, first, rows_out, 0])
            first += nblk
        self.total_blocks = first
        self._rows = rows
        self.table = None

    def _build_table(self):
        ptrs = tuple((spec[0].data_ptr(), spec[5].data_ptr() if len(spec) > 5 and spec[5] is not None else 0) for spec in self.specs)
        if ptrs != self._ptrs:
            for r, (ptr, _), spec in zip(self._rows, ptrs, self.specs):
                r[0] = ptr
                r[9] = spec[5].data_ptr() if len(spec) > 5 and spec[5] is not None else 0
            dev = self.specs[0][0].device
            self.table = torch.tensor(self._rows, dtype=torch.int64).to(dev)
            self._ptrs = ptrs

    def refresh(self, generation):
        stamp = (generation, tuple((spec[0]._version, spec[0].data_ptr(), spec[5]._version if len(spec) > 5 and spec[5] is not None else 0)
                                   for spec in self.specs))
        if stamp == self.stamp:
            return
        self._build_table()
        ops._call("pack_weights_multi", self.table.data_ptr(), len(self._rows), self.total_blocks)
        self.stamp = stamp

    def get(self, param, mode):
        return self.outputs.get((id(param), mode))

    def shared(self, name):
        """The shared operand ``name`` [rows_total][ld] (without its spare row)."""
        buf = self._shared[name]
        return buf[: buf.shape[0] - 1]


class _WeightCache:
    def __init__(self):
        self._store = {}
        self._packs = weakref.WeakKeyDictionary()  # model -> ModelPack
        self.generation = 0  # bumped by code that updates parameters behind autograd's back (fused optimizer kernels)

    def bump(self):
        self.generation += 1

    def model_pack(self, model, spec_fn):
        """Return the model's ModelPack (built on first use from spec_fn(model)), refreshed for the current parameters."""
        pack = self._packs.get(model)
        if pack is None or getattr(pack, "_spec_key", None) != spec_fn.key(model):
            pack = ModelPack(spec_fn(model))
            pack._spec_key = spec_fn.key(model)
            self._packs[model] = pack
        pack.refresh(self.generation)
        return pack

    def get(self, param, mode, ld=None, pad_rows=None, pad_cols=None):
        """The packed bf16 operand of ``param`` (ops.pack_weight ``mode``), cached until the parameter changes.  Mode 0:
        row pitch ``ld``, zero rows appended up to ``pad_rows`` (padded output channels).  Mode 1: row pitch ``pad_cols``
        (else ``ld``), zero rows appended up to ``pad_rows`` (padded input channels)."""
        key = (id(param), mode, ld, pad_rows, pad_cols)
        hit = self._store.get(key)
        stamp = (param._version, param.data_ptr(), self.generation)
        if hit is not None and hit[0] == stamp and hit[2]() is param:
            return hit[1]
        w = param.detach()
        if mode == 0:
            packed = ops.pack_weight(w, 0, ld=ld)
        else:
            packed = ops.pack_weight(w, 1, ld=pad_cols if pad_cols is not None else ld)
        if pad_rows is not None and pad_rows != packed.shape[0]:
            full = torch.zeros(pad_rows, packed.shape[1], dtype=packed.dtype, device=packed.device)
            full[: packed.shape[0]] = packed
            packed = full
        self._store[key] = (stamp, packed, weakref.ref(param))
        if len(self._store) > 4096:
            self._store = {k: v for k, v in self._store.items() if v[2]() is not None}
        return packed

    def clear(self):
        self._store.clear()
        self._packs = weakref.WeakKeyDictionary()


weight_cache = _WeightCache()
