"""Host<->device pipelining for inference over a stream of batches.

The reference pipelines (ml3d/torch/pipelines/semantic_segmentation.py:141-178 run_test,
object_detection.py:96-139 run_valid) move every batch to the device synchronously
(`inputs['data'].to(device)`) and read the result back before touching the next batch.  The
PCIe copy of a SemanticKITTI batch (~90 MB of neighbour indices) is comparable to the fused
forward, so the runner overlaps them: the inputs of batch k+1 cross PCIe on a
copy stream while batch k computes, and the result of batch k returns on a second copy
stream.  Every batch's inputs and results still cross the bus; nothing is cached.
"""
import torch


def _is_t(x):
    return isinstance(x, torch.Tensor)


def _alloc_like(x, dev):
    if _is_t(x):
        return torch.empty(x.shape, dtype=x.dtype, device=dev)
    if isinstance(x, dict):
        return {k: _alloc_like(v, dev) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_alloc_like(v, dev) for v in x]
    return x


def _same_layout(a, b):
    if _is_t(a):
        return _is_t(b) and a.shape == b.shape and a.dtype == b.dtype
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same_layout(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(_same_layout(x, y) for x, y in zip(a, b))
    return True


def _copy_tree(dst, src):
    if _is_t(src):
        dst.copy_(src, non_blocking=True)
        return dst
    if isinstance(src, dict):
        return {k: _copy_tree(dst[k], v) for k, v in src.items()}
    if isinstance(src, (list, tuple)):
        return [_copy_tree(d, s) for d, s in zip(dst, src)]
    return src   # python scalars / None travel by value


class PipelinedRunner:
    """runner = PipelinedRunner(model); for out in runner.run(batches): ...

    `batches` yields host pytrees (tensors should be pinned for the copies to overlap);
    `run` yields, in order, the model outputs as pinned host tensors (a tuple when the model
    returns several).  A yielded result stays valid until the next one is requested.  The model is called with device-resident inputs on the current stream."""

    SLOTS = 2

    def __init__(self, model, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("PipelinedRunner needs a CUDA device")
        self.model = model
        self.device = torch.device(device or getattr(model, "device", "cuda"))
        self.s_in = torch.cuda.Stream(self.device)
        self.s_out = torch.cuda.Stream(self.device)
        self._dev_in = [None] * self.SLOTS
        self._dev_out = [None] * self.SLOTS
        self._host_out = [None] * self.SLOTS

    def run(self, batches):
        main = torch.cuda.current_stream(self.device)
        in_ready = [None] * self.SLOTS    # H2D of the slot finished (recorded on s_in)
        in_free = [None] * self.SLOTS     # forward reading the slot finished (recorded on main)
        out_ready = [None] * self.SLOTS   # result staged in the slot (recorded on main)
        out_done = [None] * self.SLOTS    # D2H of the slot finished (recorded on s_out)
        pending = None
        for k, host in enumerate(batches):
            s = k % self.SLOTS
            # ---- inputs of batch k: H2D on the copy stream
            fresh = None
            if self._dev_in[s] is None or not _same_layout(self._dev_in[s], host):
                if in_free[s] is not None:
                    in_free[s].synchronize()
                self._dev_in[s] = _alloc_like(host, self.device)
                # The caching allocator hands out blocks in the order of the ALLOCATING stream (main): a recycled block
                # may still be read by kernels queued on main.  The copy stream must not write it before they are done.
                fresh = torch.cuda.Event()
                fresh.record(main)
            with torch.cuda.stream(self.s_in):
                if fresh is not None:
                    self.s_in.wait_event(fresh)
                if in_free[s] is not None:
                    self.s_in.wait_event(in_free[s])
                dev_in = _copy_tree(self._dev_in[s], host)
                in_ready[s] = torch.cuda.Event()
                in_ready[s].record(self.s_in)
            # ---- forward on the caller's stream
            main.wait_event(in_ready[s])
            out = self.model(dev_in)
            single = _is_t(out)
            outs = (out,) if single else tuple(out)
            in_free[s] = torch.cuda.Event()
            in_free[s].record(main)
            # ---- stage the result (the model may reuse its output buffers next step)
            if (self._dev_out[s] is None or len(self._dev_out[s]) != len(outs) or
                    any(d.shape != o.shape or d.dtype != o.dtype for d, o in zip(self._dev_out[s], outs))):
                if out_done[s] is not None:
                    out_done[s].synchronize()
                self._dev_out[s] = [torch.empty_like(o, memory_format=torch.contiguous_format) for o in outs]
                self._host_out[s] = [torch.empty(o.shape, dtype=o.dtype).pin_memory() for o in outs]
            if out_done[s] is not None:
                main.wait_event(out_done[s])
            for d, o in zip(self._dev_out[s], outs):
                d.copy_(o, non_blocking=True)
            out_ready[s] = torch.cuda.Event()
            out_ready[s].record(main)
            with torch.cuda.stream(self.s_out):
                self.s_out.wait_event(out_ready[s])
                for h, d in zip(self._host_out[s], self._dev_out[s]):
                    h.copy_(d, non_blocking=True)
                out_done[s] = torch.cuda.Event()
                out_done[s].record(self.s_out)
            # ---- hand back the previous batch while this one is in flight
            if pending is not None:
                ps, psingle = pending
                out_done[ps].synchronize()
                yield self._host_out[ps][0] if psingle else tuple(self._host_out[ps])
            pending = (s, single)
        if pending is not None:
            ps, psingle = pending
            out_done[ps].synchronize()
            yield self._host_out[ps][0] if psingle else tuple(self._host_out[ps])
