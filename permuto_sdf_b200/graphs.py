"""CUDA-graph capture and replay for the direct training loops (Trainer, NerfTrainer, SurfaceFit, SpaceTimeFit).

The policy: the first iteration with a given shape runs eagerly on a side stream, so that workspaces and the library's lazy state are
created there; the next one is captured and, since a capture records the work without running it, replayed once; later iterations
replay the graph while the shape key matches and the iteration stays inside the range over which the captured Python control flow holds
(DeviceIter). A captured graph writes into buffers that were allocated outside the capture, so the graph's entry holds them for as long
as it lives."""
import torch

from . import _lib


def on_stream(stream, fn, *args):
    """fn(*args) on `stream`, behind the work queued so far on the current stream; the current stream then waits for it -> fn's result"""
    cur = torch.cuda.current_stream()
    stream.wait_stream(cur)
    with torch.cuda.stream(stream):
        out = fn(*args)
    cur.wait_stream(stream)
    return out


def capture(stream, fn, *args, pool=None, count_launches=False):
    """record fn(*args) into a new CUDA graph on `stream` (nothing runs) -> (graph, fn's result, kernels of this library recorded or None).
    The count is a statistics window of its own: an outer window is paused while it is open."""
    torch.cuda.synchronize()
    if count_launches:
        paused = _lib.stats_pause()
        _lib.stats_begin(with_events=False)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream, pool=pool):
        out = fn(*args)
    launches = None
    if count_launches:
        launches = _lib.stats_end()[1]
        _lib.stats_resume(paused)
    return graph, out, launches


def graph_state(stream, *names):
    """graph-mode state of a loop: its capture stream, the number of captures so far and an empty slot per name (see run)"""
    return dict(stream=stream, captures=0, **{n: dict(graph=None, warm=None) for n in names})


def run(state, slot, key, dit, fn, inputs=(), keep=None):
    """fn(dit, *inputs) under the policy of this module -> fn's result (under replay: the result of the capture, whose buffers the graph
    rewrites). state: the loop's graph_state (capture stream and count). slot: a dict that holds one captured graph under "graph" (None
    while there is none) and the key of the last eager run under "warm". dit: the DeviceIter of this iteration. inputs: tensors (or None)
    copied into the graph's static buffers before each replay. keep: called right after a capture -> the buffers allocated outside the
    capture that the graph writes; the entry holds them for as long as it lives."""
    e = slot["graph"]
    if e is not None and e["key"] == key and e["lo"] <= int(dit) < e["hi"]:
        for dst, src in zip(e["static"], inputs):
            if dst is not None:
                dst.copy_(src, non_blocking=True)
        e["graph"].replay()
        return e["out"]
    if slot["warm"] != key:
        out = on_stream(state["stream"], fn, dit, *inputs)
        slot["warm"] = key
        return out
    static = [None if t is None else t.detach().to(dit.dev.device).clone() for t in inputs]
    graph, out, _ = capture(state["stream"], fn, dit, *static)
    slot["graph"] = dict(graph=graph, key=key, lo=dit.lo, hi=dit.hi, static=static, out=out, keep=None if keep is None else keep())
    state["captures"] += 1
    graph.replay()                     # the capture recorded the work, it did not run it
    return out


def sampler_graph_mode(on, generators):
    """the class-wide sampler state of graph mode: static-capacity ray-sample containers and the pcg32 `generators` on the device (on),
    or exactly sized containers and host generators"""
    from .permuto_sdf import RaySamplesPacked
    RaySamplesPacked.static_capacity = on
    for r in generators:
        if on:
            r.to_device()
        else:
            r.to_host()
