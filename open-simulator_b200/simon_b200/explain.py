"""Explained placement decisions on the host: Explanation, built from the engine's records (Engine.explanations, simon_explain_set),
with the reference's plugin names, FitError reason texts and klog V(10) lines (generic_scheduler.go:502-506, 558-562)."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List

import numpy as np

from . import abi
from .compiler import Compiled, _avoid_annotations, _extra_vector, _image_states

# weighted score of each device word (include/simon_gpu.h, simon_explain_node): (plugin, word, weight), in the order the reference's
# default profile lists its score plugins; word 7, the static row, is split by static_parts
PLUGINS = [("NodeResourcesBalancedAllocation", 0, 1), ("NodeResourcesLeastAllocated", 1, 1), ("InterPodAffinity", 2, 1),
           ("NodeAffinity", 3, 1), ("PodTopologySpread", 4, 2), ("TaintToleration", 5, 1), ("Simon", 6, 1),
           ("Open-Gpu-Share", 6, 1), ("Open-Local", 9, 1)]


@dataclass
class ExplainedNode:
    Name: str
    Total: int
    Scores: Dict[str, int]          # plugin -> weighted score


@dataclass
class Explanation:
    Pod: str                        # namespace/name
    Node: str                       # the node it was placed on, "" if unschedulable
    Feasible: int
    Nodes: List[ExplainedNode] = field(default_factory=list)
    Rejected: Dict[str, int] = field(default_factory=dict)      # FitError reason text -> nodes
    Reason: str = ""                # the FitError message of an unschedulable pod

    def Lines(self) -> List[str]:
        """The reference's two V(10) line formats, restricted to the listed nodes: one "Plugin <name> scores on <ns>/<pod> => [...]"
        per score plugin, then one "Host <node> => Score <total>" per node."""
        if not self.Nodes:
            return []
        out = []
        for name in self.Nodes[0].Scores:
            lst = " ".join("{%s %d}" % (n.Name, n.Scores[name]) for n in self.Nodes)
            out.append(f"Plugin {name} scores on {self.Pod} => [{lst}]")
        out += [f"Host {n.Name} => Score {n.Total}" for n in self.Nodes]
        return out


def static_parts(compiled: Compiled, cls: int, nodes, extra_plugins=None) -> List[Dict[str, int]]:
    """Word 7 of pod class `cls` on each of `nodes` split into ImageLocality, NodePreferAvoidPods (weight 10000) and each host-side
    extra score plugin (weight 0 counts as 1), from the compiler's own tables (compiler._extra_vector)."""
    N = compiled.n_nodes
    c = compiled.classes[cls]
    img = _image_states(compiled.node_objs, compiled.node_orig_index)
    avoid = _avoid_annotations(compiled.node_objs)
    vec = _extra_vector(c, img, avoid, N) if (img is not None or avoid is not None) else None
    out = []
    for g in nodes:
        v = 1000000 if vec is None else int(vec[g])         # ImageLocality 0 + 10000 x NodePreferAvoidPods 100
        d = {"ImageLocality": v % 10000, "NodePreferAvoidPods": 10000 * (v // 10000)}
        for pl in extra_plugins or []:
            w = int(pl.weight) if int(pl.weight) != 0 else 1
            d[pl.name] = w * int(pl.score(c.tmpl.pod, compiled.node_objs[g]))
        out.append(d)
    return out


def build(compiled: Compiled, pod: int, rec, nodes, extra_plugins=None) -> Explanation:
    """The Explanation of pod index `pod` from its record and node rows (Engine.explanations).  Asserts that the parts of word 7 sum to
    the device's word, and that each listed total is the sum of its weighted scores."""
    from .simulator import _static_reasons, fit_reasons, format_fit_error
    r = compiled.pod_recs[pod]
    name = f"{r.tmpl.namespace}/{r.name}"
    node = int(rec["node"])
    if node == abi.EXPLAIN_NOT_RUN:
        raise RuntimeError(f"pod {name} was not explained by the run")
    counts = np.asarray(rec["rejected"], np.uint32)
    reached = compiled.pods["pod_fixed_node"][pod] == -1 and node != -3
    ex = Explanation(Pod=name, Node=compiled.node_names[node] if node >= 0 else "", Feasible=int(rec["feasible"]))
    if not reached:
        return ex
    static = _static_reasons(compiled, r, range(compiled.n_nodes)) if counts[abi.SFC_STATIC] else {}
    ex.Rejected = fit_reasons(compiled, counts, static)
    if node == -1:
        ex.Reason = format_fit_error(compiled, r, counts)
    k = int(rec["n_top"])
    gs = [int(x["node"]) for x in nodes[:k]]
    parts = static_parts(compiled, int(compiled.pods["pod_class"][pod]), gs, extra_plugins)
    for x, g, st in zip(nodes[:k], gs, parts):
        w = [int(v) for v in x["words"]]
        scores = {p: wt * w[i] for p, i, wt in PLUGINS}
        if ex.Feasible > 1:
            assert sum(st.values()) == w[7], f"{name} on {compiled.node_names[g]}: static parts {st} do not sum to {w[7]}"
            scores.update(st)
        else:                       # one feasible node: nothing is scored
            scores.update({kk: 0 for kk in st})
        assert sum(scores.values()) == w[8], f"{name} on {compiled.node_names[g]}: scores {scores} do not sum to {w[8]}"
        ex.Nodes.append(ExplainedNode(compiled.node_names[g], w[8], scores))
    return ex


def pod_index(compiled: Compiled) -> Dict[str, int]:
    """namespace/name -> pod index of the compiled pod list."""
    return {f"{r.tmpl.namespace}/{r.name}": i for i, r in enumerate(compiled.pod_recs)}

