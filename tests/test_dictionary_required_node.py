"""yk_dict_pod_required_node: a DaemonSet pod's masks, with its affinity resolved against the node it is bound to run on.

For random nodes and pods (the generators of test_dictionary_random), "the masks pass on node n and required_node == n" must
equal "the string-level Kubernetes verdict (oracle/py_k8s_predicates.py) on n, and n is the required node".  Host code: no GPU
needed."""
import random

import pytest

from oracle import py_k8s_predicates as k8s
from yunikorn_k8shim_b200.dictionary import Dictionary
import test_dictionary_random as tdr

NONE = 0xFFFFFFFF
SLOWPATH = 1
IMPOSSIBLE = 1 << 63


def passes(m, bits, i):
    lb, tb = bits
    return (tb & ~m.tolerated_bits) == 0 and (lb & m.required_bits) == m.required_bits and (lb & m.forbidden_bits) == 0 \
        and m.required_node == i


def encode(d, name, p):
    return d.pod_required_node(name, node_selector=p.get("node_selector"), affinity_terms=p.get("affinity_terms"),
                               has_affinity=p.get("has_affinity", False), tolerations=p.get("tolerations"),
                               node_name=p.get("node_name"))


@pytest.mark.parametrize("seed", range(40))
def test_masks_give_the_string_level_verdict_on_the_required_node(seed):
    rng = random.Random(seed + 500)
    n_nodes = rng.randrange(3, 14)
    nodes = [tdr._rand_node(rng, i) for i in range(n_nodes)]
    pods = [tdr._rand_pod(rng, n_nodes) for _ in range(rng.randrange(5, 30))]
    for p in pods:   # most pods name their node through a matchFields term, as a DaemonSet's pods do
        if rng.random() < 0.7:
            p["has_affinity"] = True
            p.setdefault("affinity_terms", [])
            p["affinity_terms"].append({"expr": [tdr._rand_req(rng)] if rng.random() < 0.3 else [],
                                        "fields": [{"key": "metadata.name", "op": "In", "values": [f"node-{rng.randrange(n_nodes + 1)}"]}]})
    d = Dictionary()
    try:
        for i, nd in enumerate(nodes):
            d.node(i, nd["name"], nd["labels"], nd["taints"], nd["unschedulable"])
        names = [f"node-{rng.randrange(n_nodes + 1)}" for _ in pods]   # node-{n_nodes} is unknown
        masks = [encode(d, name, p) for name, p in zip(names, pods)]
        bits = [d.node_bits(i) for i in range(n_nodes)]
        checked = 0
        for p, name, m in zip(pods, names, masks):
            if m.flags & SLOWPATH:
                continue
            for i, nd in enumerate(nodes):
                want = k8s.fits(p, nd) and nd["name"] == name
                assert passes(m, bits[i], i) == want, (seed, name, p, nd)
                checked += 1
        assert checked > 0
    finally:
        d.close()


def daemon_pod(i):
    return dict(has_affinity=True, affinity_terms=[{"fields": [{"key": "metadata.name", "op": "In", "values": [f"node-{i}"]}]}],
                tolerations=[{"key": "node.kubernetes.io/not-ready", "op": "Exists", "effect": "NoExecute"},
                             {"key": k8s.UNSCHEDULABLE_KEY, "op": "Exists", "effect": "NoSchedule"}])


def test_a_rollout_takes_no_label_bit():
    d = Dictionary()
    try:
        for i in range(1000):
            d.node(i, f"node-{i}", {"zone": "abc"[i % 3]})
        g = d.generation
        for i in range(1000):
            m = encode(d, f"node-{i}", daemon_pod(i))
            assert m.required_bits == 0 and m.forbidden_bits == 0 and not (m.flags & SLOWPATH) and m.required_node == i
        assert d.generation == g
        # the same pods through yk_dict_pod fill the dictionary: the reason this call exists
        assert any(d.pod(**daemon_pod(i)).flags & SLOWPATH for i in range(1000))
    finally:
        d.close()


def test_unconditional_and_empty_terms():
    d = Dictionary()
    try:
        d.node(0, "node-0", {"zone": "a"})
        d.node(1, "node-1", {})
        fields = {"fields": [{"key": "metadata.name", "op": "In", "values": ["node-1"]}]}
        zone = {"expr": [{"key": "zone", "op": "In", "values": ["a"]}]}
        # a term whose fields accept node-1 and that has no expression matches it whatever its labels: no bit
        m = encode(d, "node-1", dict(has_affinity=True, affinity_terms=[zone, fields]))
        assert m.required_bits == 0 and m.required_node == 1
        # an originally empty term still matches nothing
        m = encode(d, "node-1", dict(has_affinity=True, affinity_terms=[{}]))
        assert m.required_bits & IMPOSSIBLE
        # fields that reject the node drop their term; the zone term remains and node-1 has no zone
        m = encode(d, "node-1", dict(has_affinity=True, affinity_terms=[zone, {"fields": [{"key": "metadata.name", "op": "NotIn",
                                                                                            "values": ["node-1"]}]}]))
        assert not passes(m, d.node_bits(1), 1)
        assert passes(encode(d, "node-0", dict(has_affinity=True, affinity_terms=[zone])), d.node_bits(0), 0)
    finally:
        d.close()


def test_unknown_or_conflicting_node_name():
    d = Dictionary()
    try:
        d.node(0, "node-0")
        m = encode(d, "node-9", daemon_pod(9))
        assert m.required_bits & IMPOSSIBLE and m.required_node == NONE
        m = encode(d, "node-0", dict(node_name="node-7"))
        assert m.required_bits & IMPOSSIBLE and m.required_node == 0
        m = encode(d, "node-0", dict(node_name="node-0"))
        assert m.required_bits == 0 and m.required_node == 0
    finally:
        d.close()
