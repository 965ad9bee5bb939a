"""Data-parallel gradient synchronisation for the B200 fusion block (one process per GPU, NCCL over NVLink).

Replaces the reference's torch DistributedDataParallel wrap (mmf/trainers/core/device.py:105-110) for this path:
the engine's weight-gradient GEMMs already accumulate into ONE flat fp32 buffer per encoder, so buckets are
contiguous SLICES of that buffer (no bucket copies, no find_unused_parameters graph walk - parameters the path
never touches, e.g. ViLBERT's q_dense*, are simply not in the pack).  As soon as the backward of layer l has
enqueued its last kernel, the slice holding layers >= l that has not been sent yet is all-reduced (AVG) on a
side stream, overlapping the remaining backward kernels; the end-of-backward callback joins the streams.

`mode`: "bucket" (above) or "end" - ONE all-reduce per flat buffer after the backward.  The exchange is small next to the
step (config 2: 346 MB fp32 = ~0.9 ms at the measured 725 GB/s bus bandwidth against a 29 ms step), while an NCCL kernel
that is co-scheduled with the persistent one-CTA-per-SM GEMMs (static tile schedule, 2-CTA clusters that need a whole
TPC) takes SMs away for as long as it runs and stretches every GEMM it overlaps: r1 lost 7-9 % that way at N = 2..8.
"end" gives the collective the idle machine at full bandwidth.  Both are measured by bench.py (MMFB_DDP_MODE).

Gradient accumulation: inside `no_sync()` nothing is communicated (the reference all-reduces on every micro-batch,
SURVEY.md 2.3); the final micro-batch reduces the accumulated buffer.
"""
import contextlib

import torch
import torch.distributed as dist
from torch import nn
from torch.autograd import Variable


def _runners(module):
    out = []
    for m in module.modules():
        r = getattr(m, "_runner", None)
        if r is not None and r not in out:
            out.append(r)
    return out


class B200DataParallel(nn.Module):
    def __init__(self, module, process_group=None, bucket_bytes=64 << 20, overlap=True, mode=None, payload=None):
        """payload: "fp32" (default: the flat fp32 gradient buffer is reduced as it is, the reference's DDP semantics) or
        "bf16" (the buffer is cast to bf16, reduced, and cast back: half the bytes on the wire for a 2^-9 relative rounding
        of each averaged gradient - the trade torch's bf16_compress_hook makes; opt-in)."""
        super().__init__()
        import os
        self.mode = mode or os.environ.get("MMFB_DDP_MODE", "bucket")
        self.payload = payload or os.environ.get("MMFB_DDP_PAYLOAD", "fp32")
        if self.payload not in ("fp32", "bf16"):
            raise ValueError("B200DataParallel payload must be 'fp32' or 'bf16', got %r" % (self.payload,))
        if self.mode not in ("bucket", "end"):
            raise ValueError("B200DataParallel mode must be 'bucket' or 'end', got %r" % (self.mode,))
        if not dist.is_initialized():
            raise RuntimeError("B200DataParallel needs an initialised torch.distributed process group")
        self.module = module
        self.group = process_group
        self.world = dist.get_world_size(process_group)
        self.bucket_bytes = int(bucket_bytes)
        self.overlap = overlap
        self._sync = True
        self._comm_stream = None
        self._pending = []
        self._callback_queued = False
        self._state = {}
        for r in _runners(module):
            r.grad_ready_hook = self._make_hook(r)
        # parameters that live outside the engine packs (embedding tables held by torch, heads ...)
        self._broadcast_parameters()

    def _broadcast_parameters(self):
        if self.world == 1:
            return
        for p in self.module.parameters():
            dist.broadcast(p.data, src=0, group=self.group)
        for b in self.module.buffers():
            if b.is_floating_point():
                dist.broadcast(b.data, src=0, group=self.group)

    # ---- bucket logic -----------------------------------------------------------------------------------
    def _make_hook(self, runner):
        def hook(step_index):
            if not self._sync or self.world == 1:
                return
            self._queue_finalize()
            pack = runner.pack
            st = self._state.setdefault(id(runner), {"hi": None})
            if self.mode == "end" or st.get("deferred") or self._must_defer(pack):
                # some parameter's .grad is (or will be) a tensor of its own - a weight tied to a torch-side head whose
                # gradient autograd installed first, or a bf16 pack whose .grad are cast copies: the flat slices are not
                # what the optimizer reads, and autograd may still be reading them on the main stream.  Reduce this
                # pack after the backward instead (_finalize).
                st["deferred"] = True
                return
            if pack.on_reentry is None:
                pack.on_reentry = lambda: self._reenter(runner)
            if st["hi"] is None:
                st["hi"] = pack.total
            lo = self._step_offset(runner, step_index)
            # send [lo, hi) once it is big enough, or when the first layer (lo == 0) has been reached
            if (st["hi"] - lo) * 4 >= self.bucket_bytes or lo == 0:
                self._all_reduce(pack.grad[lo:st["hi"]])
                st["hi"] = lo
        return hook

    @staticmethod
    def _aliases(pack, i):
        g = pack.params[i].grad
        return g is not None and g.dtype == torch.float32 and g.data_ptr() == pack._gptrs[i]

    @classmethod
    def _must_defer(cls, pack):
        if pack.dtype != torch.float32:
            return True
        return any(p.grad is not None and not cls._aliases(pack, i) for i, p in enumerate(pack.params))

    def _reenter(self, runner):
        """The runner backs a second autograd node of the SAME backward pass (module applied twice in the graph): its
        kernels are about to add local gradients on top of regions that were already averaged.  Let the in-flight
        all-reduces land, then send every region again as the second node completes it: the mean over ranks of
        (already-averaged part + local part) is the mean of the total, the averaged part being equal on all ranks."""
        if self._comm_stream is not None and self._pending:
            torch.cuda.current_stream().wait_stream(self._comm_stream)
            self._pending = []
        st = self._state.get(id(runner))
        if st is not None:
            st["hi"] = None

    @staticmethod
    def _step_offset(runner, step_index):
        """offset (elements) in the flat buffer where the parameters of execution step `step_index` start; the
        packs are laid out in execution order, so everything at or above it is complete once that step's backward
        has been enqueued."""
        return runner.step_offsets[step_index]

    def _avg(self, flat):
        """mean over ranks: NCCL reduces with AVG in one pass; gloo (CPU tests) has no AVG"""
        if self.payload == "bf16" and flat.dtype == torch.float32 and flat.numel() >= (1 << 16):
            wire = flat.to(torch.bfloat16)
            self._avg_raw(wire)
            flat.copy_(wire)
            return
        self._avg_raw(flat)

    def _avg_raw(self, flat):
        if dist.get_backend(self.group) == "nccl":
            dist.all_reduce(flat, op=dist.ReduceOp.AVG, group=self.group)
        else:
            dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group)
            flat.div_(self.world)

    def _all_reduce(self, flat):
        if flat.numel() == 0:
            return
        if self.overlap and flat.is_cuda:
            if self._comm_stream is None:
                self._comm_stream = torch.cuda.Stream()
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            self._comm_stream.wait_event(ev)
            with torch.cuda.stream(self._comm_stream):
                self._avg(flat)
            self._pending.append(flat)
        else:
            self._avg(flat)

    def _queue_finalize(self):
        if not self._callback_queued:
            self._callback_queued = True
            Variable._execution_engine.queue_callback(self._finalize)

    def _finalize(self):
        """end of backward: flush what the hooks have not sent, reduce non-pack gradients, join the comm stream"""
        self._callback_queued = False
        if self._sync and self.world > 1:
            for r in _runners(self.module):
                st = self._state.get(id(r))
                if st is not None and st.get("deferred"):
                    if r.pack.dtype == torch.float32:
                        self._all_reduce(r.pack.grad)          # the aliased parameters of the pack; the others go below
                    st["deferred"] = False
                elif st is not None and st["hi"] not in (None, 0):
                    self._all_reduce(r.pack.grad[0:st["hi"]])
                if st is not None:
                    st["hi"] = None
            self._reduce_loose_params()
            if self._comm_stream is not None and self._pending:
                torch.cuda.current_stream().wait_stream(self._comm_stream)
                self._pending = []

    def _reduce_loose_params(self):
        # a packed parameter counts as reduced only if its .grad IS its slice of the flat buffer; anything else (tied to a
        # torch-side head, bf16 cast copies, a grad installed by another node) is reduced here like an unpacked one
        packed = set()
        for r in _runners(self.module):
            if r.pack is not None:
                packed.update(id(p) for i, p in enumerate(r.pack.params) if self._aliases(r.pack, i))
        loose = [p for p in self.module.parameters() if id(p) not in packed and p.grad is not None]
        if not loose:
            return
        flat = torch.cat([p.grad.reshape(-1).float() for p in loose])
        self._avg(flat)
        o = 0
        for p in loose:
            n = p.numel()
            p.grad.copy_(flat[o:o + n].view_as(p.grad))
            o += n

    # ---- public surface ---------------------------------------------------------------------------------
    @contextlib.contextmanager
    def no_sync(self):
        old, self._sync = self._sync, False
        try:
            yield
        finally:
            self._sync = old

    def reduce_now(self):
        """all-reduce everything that accumulated under no_sync() (call after the last micro-batch's backward if it
        also ran under no_sync)."""
        if self.world == 1:
            return
        for r in _runners(self.module):
            if r.pack is not None and r.pack.dtype == torch.float32:
                self._avg(r.pack.grad)
        self._reduce_loose_params()

    def forward(self, *args, **kwargs):
        for r in _runners(self.module):
            self._state.pop(id(r), None)
        return self.module(*args, **kwargs)
