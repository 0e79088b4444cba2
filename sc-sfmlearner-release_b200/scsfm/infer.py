"""Inference: a network's fused eval forward (BatchNorm in the convolution epilogues, no activation record) replayed from a
CUDA graph.

    pred = Predictor(disp_net.eval())
    disp = pred(img)            # [B,1,H,W], exactly what disp_net(img) returns under torch.no_grad()
    pose = Predictor(pose_net.eval())(img1, img2)     # [B,6]

One graph is captured per input shape.  Every replay starts with the operand-mirror refresh of the weights and the eval-mode
BatchNorm prepare, so it always reads the current parameters and running statistics (ArenaAdam and the BatchNorm kernels
write through raw pointers that torch's version counters do not see: there is no staleness tracking to get wrong).  A graph
bakes in device addresses, so it is keyed on all of them: the input shape, the network's convolution context (replaced by
set_conv_mode), the parameter arena, the flipped-weight table and every BatchNorm buffer; when one changes the graph is
captured again.  At most `max_graphs` graphs are kept (least recently used dropped first): each holds a private memory
pool sized like one eval forward of its shape.  Eager execution is the plain module: net.eval() under torch.no_grad().
"""
import collections

import torch

from . import nets as N


class Predictor:
    def __init__(self, net, max_graphs=4):
        if not isinstance(net, N.ArenaNet):
            raise TypeError("Predictor takes a DispResNet or PoseResNet of this package, got %s" % type(net).__name__)
        self.net = net
        self.max_graphs = max_graphs
        self._graphs = collections.OrderedDict()
        self.captures = 0           # graphs captured so far (for tests and diagnostics)

    def _key(self, inputs):
        net = self.net
        bns = [m for m in net.modules() if isinstance(m, N.BNParams)]
        return (tuple((tuple(x.shape), x.device) for x in inputs), id(net.ctx), id(net.ctx._table), net._flat.data_ptr(),
                net._flat_tf32.data_ptr(), N.O.BnEvalTable.key_of(bns))

    def _capture(self, inputs):
        net = self.net
        self.captures += 1
        static = [torch.empty_like(x, dtype=torch.float32, memory_format=torch.contiguous_format) for x in inputs]
        for s, x in zip(static, inputs):
            s.copy_(x)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            net(*static)             # warm-up: builds the job tables and sizes the allocations outside the capture
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        net._tf32_version = None     # the operand-mirror refresh is part of every replay
        with torch.cuda.graph(graph):
            out = net(*static)
        net._tf32_version = None     # the capture did not run it: the next eager call recomputes the mirror
        # the entry keeps alive everything whose address the graph holds
        return {"graph": graph, "inputs": static, "out": out, "ctx": net.ctx, "flips": net.ctx._table,
                "bn_table": net._bn_eval}

    def __call__(self, *inputs):
        net = self.net
        if net.training:
            raise RuntimeError("Predictor runs the eval-mode forward: call net.eval() first")
        net.ensure_arena()
        with torch.no_grad():
            key = self._key(inputs)
            entry = self._graphs.get(key)
            if entry is None:
                entry = self._capture(inputs)
                key = self._key(inputs)          # the warm-up may have built the flipped-weight table
                self._graphs[key] = entry
                while len(self._graphs) > self.max_graphs:
                    self._graphs.popitem(last=False)
            self._graphs.move_to_end(key)
            for s, x in zip(entry["inputs"], inputs):
                s.copy_(x)
            entry["graph"].replay()
            return entry["out"].clone()

    @property
    def num_graphs(self):
        return len(self._graphs)
