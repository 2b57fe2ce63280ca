#!/usr/bin/env python
"""Transcribe the reference's Go table tests into JSON fixtures.

    KAI_REFERENCE=<KAI-Scheduler checkout> python tests/golden/gen_fixtures.py   # rewrites tests/golden/*.json

Reads the reference checkout (read-only) and writes small JSON files next to this script.
The tests read the fixtures only, never the reference.  Sources transcribed:

  actions/*.json          pkg/scheduler/actions/{allocate,reclaim,consolidation}/*_test.go and
                          pkg/scheduler/actions/integration_tests/{allocate,reclaim,consolidation,
                          consolidation_and_reclaim}/*_test.go  (test_utils.TestTopologyBasic tables:
                          cluster in -> node name / status per job out)
  nodepack.json           plugins/nodeplacement/nodepack_test.go, nodespread_test.go
  resource_division.json  plugins/proportion/resource_division/resource_division_test.go

Every case keeps the Go literal's field names; identifiers are resolved to their
values.  Cases using features outside the engine's scope (fractional GPUs, MIG,
GPU memory, DRA, pod/node affinity, custom scheduler conf) are kept but marked
`"supported": false` with a reason, so that the skipped set is explicit.
"""
from __future__ import annotations

import glob
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from go_literal import find_literals  # noqa: E402

REF = os.path.join(os.environ.get("KAI_REFERENCE", "."), "pkg", "scheduler")

IDENTS = {
    "constants.PriorityTrainNumber": 50,
    "constants.PriorityInteractivePreemptibleNumber": 75,
    "constants.PriorityBuildNumber": 100,
    "constants.PriorityInferenceNumber": 125,
    "common_info.NoMaxAllowedResource": -1.0,
    "commonconstants.UnlimitedResourceQuantity": -1.0,
    "enginev2alpha2.Preemptible": "preemptible",
    "enginev2alpha2.NonPreemptible": "non-preemptible",
    "v2alpha2.Preemptible": "preemptible",
    "v2alpha2.NonPreemptible": "non-preemptible",
    "node_info.MigStrategySingle": "single",
    "node_info.MigStrategyMixed": "mixed",
    "node_info.MigStrategyNone": "",
    "podgroup_info.DefaultSubGroup": "default-sub-group",
    "constants.DefaultQueuePriority": 100,
    "commonconstants.DefaultQueuePriority": 100,
    "time.Minute": 60.0,
    "time.Second": 1.0,
    "time.Hour": 3600.0,
}


def resolve(x):
    if isinstance(x, dict):
        if "__ident" in x and len(x) == 1:
            name = x["__ident"]
            if name.startswith("pod_status."):
                return name.split(".", 1)[1]
            if name in IDENTS:
                return IDENTS[name]
            return {"__ident": name}
        if "__binop" in x:
            l, r = resolve(x["l"]), resolve(x["r"])
            if isinstance(l, (int, float)) and isinstance(r, (int, float)):
                return {"*": l * r, "+": l + r, "-": l - r, "/": l / r if r else 0}[x["__binop"]]
            if isinstance(l, str) and isinstance(r, str) and x["__binop"] == "+":
                return l + r
            return {"__binop": x["__binop"], "l": l, "r": r}
        if "__call" in x:
            if x["__call"] == "jobs_fake.DefaultSubGroup":
                return {"podsets": [{"name": "default-sub-group", "min_available": resolve(x["args"][0])}]}
            if x["__call"].startswith("test_utils.Create") and len(x["args"]) == 1:
                return resolve(x["args"][0])
            if x["__call"] == "pointer.Duration" and len(x["args"]) == 1:  # seconds (IDENTS: time.Second = 1)
                return resolve(x["args"][0])
            if x["__call"] == "subgroup_info.NewSubGroupSet":
                # inline root set: NewSubGroupSet(RootSubGroupSetName, &TopologyConstraintInfo{...} | nil); the default
                # podset (minAvailable = len(Tasks)) is added by jobs_fake.BuildJobInfo (jobs.go:117-134)
                args = [resolve(a) for a in x["args"]]
                tc = args[1] if len(args) > 1 else None
                if isinstance(tc, dict) and set(tc) - {"__type"} <= {"Topology", "RequiredLevel", "PreferredLevel"}:
                    return {"podsets": [], "topology_constraint": {k: v for k, v in tc.items() if k != "__type"}}
                if tc is None or tc == {"__ident": "nil"}:
                    return {"podsets": []}
                return {"__unsupported": "inline SubGroupSet constructor"}
            return {"__call": x["__call"], "args": [resolve(a) for a in x["args"]]}
        if "__func" in x:
            return parse_subgroup_func(x["__func"])
        return {k: resolve(v) for k, v in x.items()}
    if isinstance(x, list):
        return [resolve(v) for v in x]
    return x


_CONSTRAINT = r'(nil|& topology_info \. TopologyConstraintInfo \{ (?:[^{}]* )?\})'
_NEWSET = re.compile(r'(\w+) : = subgroup_info \. NewSubGroupSet \( ((?:"[^"]*")|(?:subgroup_info \. RootSubGroupSetName)) , ' + _CONSTRAINT + r'(?: ,)? \)')
_ADDPODSET = re.compile(r'(\w+) \. AddPodSet \( subgroup_info \. NewPodSet \( "([^"]+)" , (\d+) , ' + _CONSTRAINT + r'(?: ,)? \) \)')
_ADDGROUP = re.compile(r'(\w+) \. AddSubGroup \( (\w+) \)')
_RETURN = re.compile(r'return (\w+) \}')
_KV = re.compile(r'(\w+) : "([^"]*)"')


def _constraint(txt):
    if txt.strip() == "nil":
        return None
    return {k: v for k, v in _KV.findall(txt)}


def parse_subgroup_func(body: str):
    """RootSubGroupSet: func() *SubGroupSet { x := NewSubGroupSet(name, constraint); x.AddPodSet(NewPodSet(name, min,
    constraint)); root.AddSubGroup(x); ...; return root } -> the SubGroupSet tree."""
    sets = {}
    events = []
    for m in _NEWSET.finditer(body):
        name = "root" if "RootSubGroupSetName" in m.group(2) else m.group(2).strip('"')
        events.append((m.start(), "set", m.group(1), name, _constraint(m.group(3))))
    for m in _ADDPODSET.finditer(body):
        events.append((m.start(), "podset", m.group(1), m.group(2), int(m.group(3)), _constraint(m.group(4))))
    for m in _ADDGROUP.finditer(body):
        events.append((m.start(), "group", m.group(1), m.group(2)))
    ret = _RETURN.search(body)
    n_stmt = body.count(": =") + body.count(". AddPodSet") + body.count(". AddSubGroup")
    if not ret or len(events) != n_stmt:
        return {"podsets": [], "__unsupported": "unparsed RootSubGroupSet"}
    for ev in sorted(events):
        if ev[1] == "set":
            sets[ev[2]] = {"name": ev[3], "constraint": ev[4], "podsets": [], "groups": []}
        elif ev[1] == "podset":
            sets[ev[2]]["podsets"].append({"name": ev[3], "min_available": ev[4], "constraint": ev[5]})
        else:
            sets[ev[2]]["groups"].append(sets[ev[3]])
    root = sets[ret.group(1)]

    def flat(g):
        out = list(g["podsets"])
        for c in g["groups"]:
            out += flat(c)
        return out

    simple = not root["groups"] and root["constraint"] is None and all(p["constraint"] is None for p in root["podsets"])
    out = {"podsets": [{"name": p["name"], "min_available": p["min_available"]} for p in flat(root)]}
    if not simple:
        out["tree"] = root
    return out


def find_unresolved(x, path=""):
    out = []
    if isinstance(x, dict):
        for k in ("__ident", "__call", "__unsupported", "__binop", "__neg"):
            if k in x:
                out.append(f"{path}:{k}={x[k] if not isinstance(x[k], (dict, list)) else '...'}")
        for k, v in x.items():
            out += find_unresolved(v, f"{path}.{k}")
    elif isinstance(x, list):
        for i, v in enumerate(x):
            out += find_unresolved(v, f"{path}[{i}]")
    return out


def evenly_distributed_topology_nodes(zones, spines_per_zone, racks_per_spine, nodes_per_rack, gpus_per_node):
    """What allocateTopology_test.go's helper buildEvenlyDistributedTopologyNodes (:3162-3188) returns: node<i> in
    creation order, labelled zone<z> / spine<global index> / rack<global index>."""
    nodes, node_id = {}, 0
    for z in range(1, zones + 1):
        for sp in range(1, spines_per_zone + 1):
            spine = sp + (z - 1) * spines_per_zone
            for r in range(1, racks_per_spine + 1):
                rack = r + (sp - 1) * racks_per_spine + (z - 1) * spines_per_zone * racks_per_spine
                for _ in range(nodes_per_rack):
                    nodes[f"node{node_id}"] = {"GPUs": gpus_per_node, "Labels": {
                        "k8s.io/zone": f"zone{z}", "k8s.io/spine": f"spine{spine}", "k8s.io/rack": f"rack{rack}"}}
                    node_id += 1
    return nodes


def normalise(topo: dict) -> dict:
    """Evaluate the two non-literal constructs the action tables use; returns the table's config overrides."""
    config = {}
    nodes = topo.get("Nodes")
    if isinstance(nodes, dict) and nodes.get("__call") == "buildEvenlyDistributedTopologyNodes":
        topo["Nodes"] = evenly_distributed_topology_nodes(*[int(a) for a in nodes["args"]])
    if isinstance(topo.get("Nodes"), dict):
        for name, node in topo["Nodes"].items():
            if node == []:  # `"node-1": {}` — an empty TestNodeBasic literal
                topo["Nodes"][name] = {}
    mocks = topo.get("Mocks")
    conf = mocks.get("SchedulerConf") if isinstance(mocks, dict) else None
    if isinstance(conf, dict):
        # a SchedulerConf that only sets the nodeplacement strategies (allocate_test.go:1306-1322) maps onto kai_config;
        # the other plugins of the default tier do not change such a table's outcome
        plugins = [p for t in conf.get("Tiers") or [] for p in t.get("Plugins") or []]
        if len(plugins) == 1 and plugins[0].get("Name") == "nodeplacement":
            strategy = {"constants.SpreadStrategy": "spread", "constants.BinpackStrategy": "binpack"}
            keys = {"constants.GPUResource": "gpu_placement", "constants.CPUResource": "cpu_placement"}
            args = plugins[0].get("Arguments") or {}
            if all(k in keys and isinstance(v, dict) and v.get("__ident") in strategy for k, v in args.items()):
                config = {keys[k]: strategy[v["__ident"]] for k, v in args.items()}
                del mocks["SchedulerConf"]
    return config


def classify(topo: dict) -> str | None:
    """Return a skip reason if the case uses features outside the engine's scope, else None."""
    for tp in topo.get("Topologies") or []:
        if not (isinstance(tp, dict) and (tp.get("Spec") or {}).get("Levels")):
            return "topology CR without levels"
    mocks = topo.get("Mocks") or {}
    if isinstance(mocks, dict) and mocks.get("SchedulerConf"):
        return "custom SchedulerConf"
    if isinstance(mocks, dict) and mocks.get("GPUMetric"):
        return "GPU metric mocks"
    for key in ("TestDRAObjects", "ResourceClaims", "ResourceSlices", "DeviceClasses"):
        if topo.get(key):
            return "DRA objects"
    if not isinstance(topo.get("Nodes") or {}, dict):
        return "nodes built by code"
    for name, node in (topo.get("Nodes") or {}).items():
        if not isinstance(node, dict):
            return "node built by code"
        if node.get("MigStrategy") or node.get("MigInstances"):
            return "MIG node"
        if node.get("GpuMemorySynced") is not None or node.get("GPUMemory"):
            return "GPU memory"
        if node.get("Labels") and not topo.get("Topologies"):
            return "node labels"
    for job in topo.get("Jobs") or []:
        g = job.get("RequiredGPUsPerTask", 0) or 0
        if float(g) != int(g):
            return "fractional GPU"
        if job.get("RequiredGpuMemory") or job.get("RequiredMultiFractionDevicesPerTask"):
            return "GPU memory / multi-fraction"
        if job.get("DeleteJobInTest"):
            return "deletion in test"
        for t in job.get("Tasks") or []:
            for k in ("PodAffinityLabels", "PodAffinityTopologyKey",
                      "PodAntiAffinityTopologyKey", "RequiredMigInstances", "IsLegacyMigTask",
                      "ResourceClaimTemplates", "ResourceClaimNames", "GPUGroups"):
                if t.get(k):
                    return f"task {k}"
    for q in topo.get("Queues") or []:
        if q.get("V1") or q.get("UseOnlyFreeCPUResources") or q.get("InteractiveTimeoutInMinutes"):
            return "legacy queue fields"
    unresolved = find_unresolved(topo)
    if unresolved:
        return "unresolved: " + "; ".join(unresolved[:3])
    return None


ACTION_SUITES = [
    # (glob relative to actions/, action list run by the reference's test driver)
    ("allocate/allocate_test.go", ["allocate"]),
    ("allocate/allocateGang_test.go", ["allocate"]),
    ("allocate/allocateElastic_test.go", ["allocate"]),
    ("allocate/allocate_subgroups_test.go", ["allocate"]),
    ("allocate/allocateTopology_test.go", ["allocate"]),
    ("reclaim/reclaim_test.go", ["reclaim"]),
    ("reclaim/reclaimGang_test.go", ["reclaim"]),
    ("reclaim/reclaimDepartments_test.go", ["reclaim"]),
    ("reclaim/reclaim_elastic_test.go", ["reclaim"]),
    ("reclaim/reclaim_sub_group_test.go", ["reclaim"]),
    ("consolidation/consolidation_test.go", ["consolidation"]),
    ("consolidation/consolidation_subgroups_test.go", ["consolidation"]),
    ("preempt/preempt_test.go", ["preempt"]),
    ("preempt/preemptGang_test.go", ["preempt"]),
    ("preempt/preempt_elastic_test.go", ["preempt"]),
    ("preempt/preempt_subgroups_test.go", ["preempt"]),
    # the driver overrides the grace period: ssn.OverrideGlobalDefaultStalenessGracePeriod(60 * time.Second) (:407)
    ("stalegangeviction/stalegangeviction_test.go", ["stalegangeviction"]),
    # integration tables run the whole default action list for several rounds
    ("integration_tests/allocate/allocate_test.go", ["allocate", "consolidation", "reclaim", "preempt", "stalegangeviction"]),
    ("integration_tests/reclaim/reclaim_test.go", ["allocate", "consolidation", "reclaim", "preempt", "stalegangeviction"]),
    ("integration_tests/consolidation/consolidation_test.go", ["allocate", "consolidation", "reclaim", "preempt", "stalegangeviction"]),
    ("integration_tests/consolidation_and_reclaim/consolidation_and_reclaim_test.go",
     ["allocate", "consolidation", "reclaim", "preempt", "stalegangeviction"]),
]


def gen_actions():
    os.makedirs(os.path.join(HERE, "actions"), exist_ok=True)
    summary = {}
    for rel, actions in ACTION_SUITES:
        path = os.path.join(REF, "actions", rel)
        src = open(path).read()
        if "preemptGang" in rel:
            # this file builds one flaky-scenario table with a Go for-loop (statements, not literals): only the
            # literal tables before it are transcribed
            cut = src.find("flaky scenario")
            if cut > 0:
                src = src[:src.rfind("func ", 0, cut)]
        # integration tables wrap the topology in TestTopologyMetadata{TestTopologyBasic: ..., RoundsUntilMatch: n}
        rounds = {}
        metas = find_literals(src, "integration_tests_utils.TestTopologyMetadata") if "TestTopologyMetadata" in src else []
        # find_literals returns the outermost `[]TestTopologyMetadata{...}` slice literal first; flatten
        flat = []
        for m in metas:
            if isinstance(m, list):
                flat += m
            else:
                flat.append(m)
        cases = []
        if flat and all(isinstance(m, dict) and "TestTopologyBasic" in m for m in flat):
            for m in flat:
                m = resolve(m)
                topo = m["TestTopologyBasic"]
                cases.append((topo, m.get("RoundsUntilMatch"), m.get("RoundsAfterMatch")))
        else:
            for topo in find_literals(src, "test_utils.TestTopologyBasic"):
                cases.append((resolve(topo), None, None))
        out = []
        wrapper_names = re.findall(r'^\t\t\tname:\s*"([^"]*)"', src, flags=re.M)
        for i, (topo, r_until, r_after) in enumerate(cases):
            topo.pop("__type", None)
            config = normalise(topo)
            if rel.startswith("stalegangeviction/"):
                config["staleness_grace_period_s"] = 60
                topo.setdefault("Name", wrapper_names[i])  # the table keeps the name beside the topology (`name:`)
            reason = classify(topo)
            out.append({
                "source": f"pkg/scheduler/actions/{rel}",
                "index": i,
                "name": topo.get("Name", ""),
                "actions": actions,
                "rounds_until_match": r_until,
                "rounds_after_match": r_after,
                "supported": reason is None,
                "skip_reason": reason,
                "config": config,
                "topology": topo,
            })
        name = rel.replace("/", "__").replace("_test.go", "") + ".json"
        with open(os.path.join(HERE, "actions", name), "w") as f:
            json.dump(out, f, indent=1, sort_keys=True)
        summary[rel] = (len(out), sum(1 for c in out if c["supported"]))
    return summary


def main():
    s = gen_actions()
    for k, (n, ok) in s.items():
        print(f"{k}: {n} cases, {ok} in scope")


if __name__ == "__main__":
    main()


# ---------------------------------------------------------------------------------------------
# unit-level known answers
# ---------------------------------------------------------------------------------------------
def _num(x, env=None):
    """Evaluate a resolved literal value to a float (constants, float64(..), simple arithmetic)."""
    env = env or {}
    if isinstance(x, bool):
        return x
    if isinstance(x, (int, float)):
        return float(x)
    if isinstance(x, str):
        return float(x)
    if isinstance(x, dict):
        if "__ident" in x:
            name = x["__ident"]
            table = {"scores.MaxHighDensity": 9.0, "commonconstants.UnlimitedResourceQuantity": -1.0,
                     "constants.UnlimitedResourceQuantity": -1.0,
                     "resource_info.MinMemory": 10.0 * 1024 * 1024}  # api/resource_info/base_resources.go:18
            if name in table:
                return table[name]
            if name in env:
                return env[name]
            raise ValueError(f"unknown identifier {name}")
        if "__binop" in x:
            l, r = _num(x["l"], env), _num(x["r"], env)
            return {"*": l * r, "+": l + r, "-": l - r, "/": l / r}[x["__binop"]]
        if "__neg" in x:
            return -_num(x["__neg"], env)
        if "__call" in x and x["__call"] in ("float64", "float32", "int", "int64") and len(x["args"]) == 1:
            return _num(x["args"][0], env)
    raise ValueError(f"cannot evaluate {x!r}")


def gen_nodeplacement():
    """plugins/nodeplacement/nodepack_test.go + nodespread_test.go: exact expected f64 scores per node."""
    out = {}
    for fname, kind in (("nodepack_test.go", "binpack"),):
        src = open(os.path.join(REF, "plugins", "nodeplacement", fname)).read()
        tables = find_literals(src, "[]testTopologyMetadata")
        found = []

        def collect(x):
            if isinstance(x, dict):
                if "testNodeMetadataMap" in x:
                    found.append(x)
                else:
                    for v in x.values():
                        collect(v)
            elif isinstance(x, list):
                for v in x:
                    collect(v)

        collect(tables)
        cases = []
        for table in [found]:
            for c in table:
                nodes = {}
                for name, nd in c["testNodeMetadataMap"].items():
                    nodes[name] = {
                        "allocatable_gpus": float(nd["nodeAllocatableGPUs"]),
                        "idle_gpus": float(nd["nodeIdleGPUs"]),
                        "expected_score": _num(nd["nodeExpectedScore"]),
                    }
                cases.append({"source": f"pkg/scheduler/plugins/nodeplacement/{fname}", "name": c["name"],
                              "task": c.get("taskName", ""), "nodes": nodes})
        out[kind] = cases
    # nodespread_test.go: anonymous-struct case lists {gpuCount|cpuMillis.., nonAllocated, expected}
    src = open(os.path.join(REF, "plugins", "nodeplacement", "nodespread_test.go")).read()
    spread = []
    for m in re.finditer(r"\{\s*(\w+):\s*([-\d.]+),\s*nonAllocated:\s*([-\d.]+),\s*expected:\s*([-\d.]+),\s*\}", src):
        spread.append({"source": "pkg/scheduler/plugins/nodeplacement/nodespread_test.go", "count_field": m.group(1),
                       "count": float(m.group(2)), "non_allocated": float(m.group(3)), "expected_score": float(m.group(4))})
    out["spread"] = spread
    with open(os.path.join(HERE, "nodeplacement.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    return {k: len(v) for k, v in out.items()}


def gen_resource_division():
    """plugins/proportion/resource_division/resource_division_test.go — the `DescribeTable("two queues", ...)`
    entries (setResourceShare on GPU with per-entry overrides) transcribed as data."""
    src = open(os.path.join(REF, "plugins", "proportion", "resource_division", "resource_division_test.go")).read()
    i = src.index('Context("two queues", func() {')
    j = src.index('It("divides the remainder even when using priorities"', i)
    block = src[i:j]
    base = find_literals(block, "map[common_info.QueueID]*rs.QueueAttributes")[0]
    if isinstance(base, list):  # `func() map[..]..{ return map[..]..{...} }` parses as [return, {...}]
        base = [x for x in base if isinstance(x, dict) and "__ident" not in x][0]
    entries = find_literals(block, "testMetadata")
    cases = []
    names = re.findall(r'Entry\("([^"]+)",\s*testMetadata', block)
    for name, e in zip(names, entries):
        queues = {}
        for qid, q in base.items():
            g = q["QueueResourceShare"]["GPU"]
            queues[qid] = {"deserved": _num(g["Deserved"]), "fair_share": _num(g["FairShare"]),
                           "oqw": _num(g["OverQuotaWeight"]), "max_allowed": _num(g["MaxAllowed"]),
                           "allocated": _num(g["Allocated"]), "request": _num(g["Request"]), "priority": 0}
        for qid, v in (e.get("maxAllowed") or {}).items():
            queues[qid]["max_allowed"] = _num(v)
        for qid, v in (e.get("gpuOverQuotaWeights") or {}).items():
            queues[qid]["oqw"] = _num(v)
        for qid, v in (e.get("request") or {}).items():
            queues[qid]["request"] = _num(v)
        for qid, v in (e.get("overQuotaPriority") or {}).items():
            queues[qid]["priority"] = int(_num(v))
        cases.append({
            "source": "pkg/scheduler/plugins/proportion/resource_division/resource_division_test.go (two queues table)",
            "name": name, "total": _num(e["totalGPUs"]), "k_value": 0.0, "queues": queues,
            "expected_remaining": _num(e.get("expectedRemaining", 0)),
            "expected_share": {k: _num(v) for k, v in (e.get("expectedShare") or {}).items()},
        })
    with open(os.path.join(HERE, "resource_division.json"), "w") as f:
        json.dump(cases, f, indent=1, sort_keys=True)
    return len(cases)


if __name__ == "__main__":
    print("nodeplacement:", gen_nodeplacement())
    print("resource_division two-queues table:", gen_resource_division())


def gen_can_reclaim():
    """plugins/proportion/reclaimable/reclaimable_test.go:34-531 — the two literal tables of `CanReclaimResources`
    (preemptible and non-preemptible reclaimer) -> tests/golden/can_reclaim_resources.json."""
    import re
    path = os.path.join(REF, "plugins", "proportion", "reclaimable", "reclaimable_test.go")
    src = open(path).read()
    blk = src[src.index('var _ = Describe("Can Reclaim Resources"'):src.index('var _ = Describe("Reclaimable - Single department"')]
    infos = find_literals(blk, "ReclaimerInfo")
    queues = [q for q in find_literals(blk, "rs.QueueAttributes") if isinstance(q, dict) and "QueueResourceShare" in q]
    expected = re.findall(r'canReclaim:\s*(true|false)', blk)
    names = re.findall(r'\bname:\s*"([^"]*)"', blk)
    assert len(infos) == len(queues) == len(expected) == len(names)
    out = []
    for name, info, queue, exp in zip(names, infos, queues, expected):
        req = [_num(a) for a in info["RequiredResources"]["args"]]  # NewResource(milliCPU, memory, gpus)
        share = {}
        for res in ("CPU", "Memory", "GPU"):
            rs_ = queue["QueueResourceShare"].get(res) or {}
            share[res] = {k: _num(rs_.get(k, 0)) for k in ("Deserved", "FairShare", "Allocated", "AllocatedNotPreemptible")}
        out.append({"name": name, "req": req, "preemptible": bool(info.get("IsPreemptable", False)), "share": share,
                    "can_reclaim": exp == "true"})
    with open(os.path.join(HERE, "can_reclaim_resources.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    return len(out)


if __name__ == "__main__":
    print("can_reclaim_resources:", gen_can_reclaim())


def gen_set_resources_share():
    """plugins/proportion/resource_division/resource_division_test.go:1111-2020 — the data-driven `SetResourcesShare`
    table (contexts x cases; three resources per queue) -> tests/golden/set_resources_share.json."""
    path = os.path.join(REF, "plugins", "proportion", "resource_division", "resource_division_test.go")
    src = open(path).read()
    blk = src[src.index('tests := map[string]map[string]struct {'):src.index('for contextName, contextData := range tests')]
    # give the anonymous struct type a name so that the literal parser sees a typed composite literal
    blk = 'tests := map[string]map[string]caseT' + blk[blk.index('}{') + 1:]
    top = find_literals(blk, 'map[string]map[string]caseT')[0]
    fields = ("Deserved", "FairShare", "OverQuotaWeight", "MaxAllowed", "Allocated", "Request")
    out = []
    for ctx, cases in top.items():
        if ctx.startswith("__"):
            continue
        for name, case in cases.items():
            if name.startswith("__"):
                continue
            queues = {}
            for qid, q in case["queues"].items():
                if qid.startswith("__"):
                    continue
                share = q.get("QueueResourceShare") or {}
                queues[qid] = {"priority": int(_num(q.get("Priority", 0))),
                               **{res: {f: _num((share.get(res) or {}).get(f, 0)) for f in fields} for res in ("GPU", "CPU", "Memory")}}
            total = {k.split(".")[-1]: _num(v) for k, v in case["totalResources"].items() if not k.startswith("__")}
            expected = {qid: {res: _num(((q.get("QueueResourceShare") or {}).get(res) or {}).get("FairShare", 0))
                              for res in ("GPU", "CPU", "Memory")}
                        for qid, q in case["expectedShare"].items() if not qid.startswith("__")}
            out.append({"context": ctx, "name": name, "queues": queues, "total": total, "expected": expected})
    with open(os.path.join(HERE, "set_resources_share.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    return len(out)


if __name__ == "__main__":
    print("set_resources_share:", gen_set_resources_share())


def gen_reclaim_strategies():
    """plugins/proportion/reclaimable/strategies/strategies_test.go:22-806 — the three literal tables (MaintainFairShare,
    MaintainFairShare multi-resource, GuaranteeDeservedQuota) -> tests/golden/reclaim_strategies.json."""
    path = os.path.join(REF, "plugins", "proportion", "reclaimable", "strategies", "strategies_test.go")
    src = open(path).read()
    fields = ("Deserved", "FairShare", "Allocated", "AllocatedNotPreemptible", "MaxAllowed")

    def queue(q):
        share = (q or {}).get("QueueResourceShare") or {}
        return {res: {f: _num((share.get(res) or {}).get(f, 0)) for f in fields} for res in ("CPU", "Memory", "GPU")}

    out = []
    pos = 0
    for ctx in ("Maintain Fair Share Strategy", "Maintain Fair Share Strategy - Multi Resource", "Guarantee Deserved Quota Strategy"):
        a = src.index(f'Context("{ctx}"', pos)
        a = src.index("tests := map[string]struct {", a)
        b = src.index("strategy := &", a)
        pos = b
        blk = src[a:b]
        blk = "tests := map[string]caseT" + blk[blk.index("}{") + 1:]
        table = find_literals(blk, "map[string]caseT")[0]
        for name, case in table.items():
            if name.startswith("__"):
                continue
            rec = {"context": ctx, "name": name, "reclaimer": queue(case.get("reclaimerQueue")),
                   "reclaimee": queue(case.get("reclaimeeQueue")), "expected": bool(case["expected"])}
            if case.get("remainingResourceShare") is not None:
                rec["remaining"] = {k.split(".")[-1]: _num(v) for k, v in case["remainingResourceShare"].items() if not k.startswith("__")}
            if case.get("reclaimerResources") is not None:
                rec["reclaimer_req"] = [_num(x) for x in case["reclaimerResources"]["args"]]
            out.append(rec)
    with open(os.path.join(HERE, "reclaim_strategies.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    return len(out)


if __name__ == "__main__":
    print("reclaim_strategies:", gen_reclaim_strategies())


def gen_capacity_policy():
    """plugins/proportion/capacity_policy/capacity_policy_test.go:24-1080 — the four literal tables (IsJobOverQueueCapacity
    x2, IsNonPreemptibleJobOverQuota, IsTaskAllocationOnNodeOverCapacity) -> tests/golden/capacity_policy.json."""
    path = os.path.join(REF, "plugins", "proportion", "capacity_policy", "capacity_policy_test.go")
    src = open(path).read()
    # `NewPodSet(..).WithPodInfos(map)` is a method chain the literal parser does not read: fold it into one call
    src = re.sub(r'subgroup_info\.NewPodSet\(([^()]*)\)\.\s*WithPodInfos\(', r'podsetWithPods(\1, ', src)
    fields = ("Deserved", "FairShare", "Allocated", "AllocatedNotPreemptible", "MaxAllowed")
    modes = ["IsJobOverQueueCapacity", "IsJobOverQueueCapacity", "IsNonPreemptibleJobOverQuota", "IsTaskAllocationOnNodeOverCapacity"]
    out, pos = [], 0
    for mode in modes:
        a = src.index("tests := map[string]struct {", pos)
        b = src.index("for name, data := range tests", a)
        pos = b
        blk = src[a:b]
        table = find_literals("tests := map[string]caseT" + blk[blk.index("}{") + 1:], "map[string]caseT")[0]
        for name, case in table.items():
            if name.startswith("__"):
                continue
            queues = {}
            for qid, q in case["queues"].items():
                if qid.startswith("__"):
                    continue
                share = q.get("QueueResourceShare") or {}
                queues[qid] = {"parent": q.get("ParentQueue", ""),
                               **{res: {f: _num((share.get(res) or {}).get(f, 0)) for f in fields} for res in ("CPU", "Memory", "GPU")}}
            job = case["job"]
            pods = list(job["PodSets"].values())[0]["args"][3]
            req = [0.0, 0.0, 0.0]  # (cpu, memory, gpu) summed over the pending pods = getRequiredQuota
            for pid, pod in pods.items():
                if pid.startswith("__") or (pod.get("Status") or {}).get("__ident") != "pod_status.Pending":
                    continue
                rr = pod["ResReq"]
                if rr["__call"].endswith("NewResourceRequirementsWithGpus"):
                    req[2] += _num(rr["args"][0])
                else:  # NewResourceRequirements(gpus, milliCpus, memory)
                    req[2] += _num(rr["args"][0])
                    req[0] += _num(rr["args"][1])
                    req[1] += _num(rr["args"][2])
            pre = (job.get("Preemptibility") or {}).get("__ident", "")
            out.append({"function": mode, "name": name, "queues": queues, "queue": job["Queue"], "req": req,
                        # PodGroupInfo.IsPreemptibleJob(): the zero value of Preemptibility is not "preemptible"
                        "preemptible": pre.endswith(".Preemptible"), "schedulable": bool(case["expectedResult"])})
    with open(os.path.join(HERE, "capacity_policy.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    return len(out)


if __name__ == "__main__":
    print("capacity_policy:", gen_capacity_policy())


def gen_capacity_checks():
    """plugins/proportion/capacity_policy/max_allowed_check_test.go:38-208 (isOverLimit), :211-459 (resultsOverLimit) and
    quota_check_test.go:32-130 (isAllocatedNonPreemptibleOverQuota), :132-338 (resultsWithNonPreemptibleOverQuota) ->
    tests/golden/capacity_checks.json, in the schema of capacity_policy.json (`req` is the table's requested share)."""
    fields = ("Deserved", "FairShare", "Allocated", "AllocatedNotPreemptible", "MaxAllowed")
    res_key = {"rs.CpuResource": "CPU", "rs.MemoryResource": "Memory", "rs.GpuResource": "GPU"}

    def quantities(m):
        m = resolve(m) if m else {}
        return {res_key[k]: _num(v) for k, v in m.items() if k in res_key}

    def tables(fname):
        src = open(os.path.join(REF, "plugins", "proportion", "capacity_policy", fname)).read()
        pos = 0
        while True:
            a = src.find("tests := map[string]struct {", pos)
            if a < 0:
                return
            b = src.index("for name, data := range tests", a)
            pos = b
            blk = src[a:b]
            yield find_literals("tests := map[string]caseT" + blk[blk.index("}{") + 1:], "map[string]caseT")[0]

    out = []
    for fname, flat_fn, tree_fn in (("max_allowed_check_test.go", "isOverLimit", "resultsOverLimit"),
                                    ("quota_check_test.go", "isAllocatedNonPreemptibleOverQuota", "resultsWithNonPreemptibleOverQuota")):
        flat, tree = list(tables(fname))
        limit = flat_fn == "isOverLimit"
        for name, case in flat.items():
            if name.startswith("__"):
                continue
            # the Ginkgo body writes two fields of one queue's shares (EmptyResource() otherwise) and calls the check
            a = quantities(case.get("maxAllowed" if limit else "deserved"))
            b = quantities(case.get("allocated" if limit else "allocatedNonPreemptible"))
            share = {res: {f: 0.0 for f in fields} for res in ("CPU", "Memory", "GPU")}
            for res in share:
                share[res]["MaxAllowed" if limit else "Deserved"] = a.get(res, 0.0)
                share[res]["Allocated" if limit else "AllocatedNotPreemptible"] = b.get(res, 0.0)
                if not limit:
                    share[res]["MaxAllowed"] = -1.0
            req = quantities(case.get("requestedQuota"))
            over = bool(case.get("isOverMaxAllowed" if limit else "expectedResult"))
            out.append({"function": flat_fn, "name": name, "queues": {"queue": {"parent": "", **share}}, "queue": "queue",
                        "req": [req.get("CPU", 0.0), req.get("Memory", 0.0), req.get("GPU", 0.0)],
                        "preemptible": limit, "schedulable": not over})
        for name, case in tree.items():
            if name.startswith("__"):
                continue
            queues = {}
            for qid, q in case["queues"].items():
                if qid.startswith("__"):
                    continue
                sh = q.get("QueueResourceShare") or {}
                queues[qid] = {"parent": q.get("ParentQueue", ""),
                               **{res: {f: _num(resolve((sh.get(res) or {}).get(f, 0))) for f in fields} for res in ("CPU", "Memory", "GPU")}}
            job = case["job"]
            req = quantities(case.get("requestedShare"))
            pre = (job.get("Preemptibility") or {}).get("__ident", "")
            out.append({"function": tree_fn, "name": name, "queues": queues, "queue": job["Queue"],
                        "req": [req.get("CPU", 0.0), req.get("Memory", 0.0), req.get("GPU", 0.0)],
                        # resultsOverLimit does not look at preemptibility; the quota check returns early for a preemptible job
                        "preemptible": True if limit else pre.endswith(".Preemptible"), "schedulable": bool(case["expectedResult"])})
    with open(os.path.join(HERE, "capacity_checks.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    return len(out)


if __name__ == "__main__":
    print("capacity_checks:", gen_capacity_checks())
