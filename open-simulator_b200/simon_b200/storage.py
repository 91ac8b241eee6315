"""Open-Local volumes (pkg/simulator/plugin/open-local.go:51-254), host side: the storage columns of include/simon_gpu.h
(simon_storage, simon_devices), and an object-level restatement of the plugin's VG and device choice that formats the failure
texts and the node annotations Bind writes.  OL = vendor/github.com/alibaba/open-local/pkg of the reference tree.

Determinism: the reference sorts the VGs of a node with an unstable sort over Go map order, so equal free sizes are taken in a
random order.  Here VGs of equal free size are taken in the order of the annotation's "vgs" list (a stable sort), the "last VG"
of an InsufficientLVMError is the last one in that order, and ScoreLVM sums over VGs in annotation order.  Free devices of equal
capacity are likewise taken in the order of the annotation's "devices" list.  Each such result is one of the reference's
possible outcomes.

Device PVCs are the volumes whose StorageClass is not one of the two LVM classes (GetPodLocalPVCs, pkg/utils/utils.go:565-623).
DividePVCAccordingToMediaType (OL/scheduler/algorithm/algo/common.go:247-260) splits them by the class's mediaType into SSD and
HDD; a missing class or any other media type drops the PVC.  Dropped PVCs only require the node annotation.  SSD and HDD PVCs
each take one free device of their media type (ProcessDevicePVC, common.go:394-448); they are placed only with the devices
opt-in (compile_storage(devices=True)), and refused with StorageError without it.  ScoreDevice of a class whose device PVCs were
all dropped is 0/0 (int(NaN) = MinInt64 on amd64): it shifts every feasible node's raw score by the same amount, which
NormalizeScore cancels.
"""
from __future__ import annotations

import json
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import objects as O
from .abi import MAX_DEV_VOLS, MAX_DEVS, MAX_VGS, MAX_VOLS

LVM_SC = ("open-local-lvm", "yoda-lvm-default")      # pkg/utils/utils.go:603 (OpenLocalSCNameLVM, YodaSCNameLVM)
MEDIA = ("ssd", "hdd")     # OL/types.go:72-73, in the order ProcessDevicePVC takes them
INT64_MIN = -(1 << 63)


class StorageError(ValueError):
    """Input the engine refuses rather than narrows (raised as compiler.CompileError by the compiler)."""


def binary_si(x: int) -> str:
    """resource.NewQuantity(x, BinarySI).String() for int64 x (vendor/k8s.io/apimachinery/pkg/api/resource/quantity.go:
    CanonicalizeBytes, amount.go AsCanonicalBase1024Bytes, suffix.go): |x| < 1024 prints as a decimal integer, otherwise the
    largest power of 1024 that divides x becomes the suffix Ki .. Ei."""
    if -1024 < x < 1024:
        return str(x)
    e = 0
    while x != 0 and x % 1024 == 0 and e < 6:
        x //= 1024
        e += 1
    return str(x) + ("", "Ki", "Mi", "Gi", "Ti", "Pi", "Ei")[e]


def _go_int_string(v, what: str) -> int:
    # encoding/json `,string` int64: a JSON string holding a decimal integer in int64 range
    if not isinstance(v, str):
        raise StorageError(f"{what}: expected a quoted integer, got {v!r}")
    try:
        n = int(v, 10)
    except ValueError:
        raise StorageError(f"{what}: {v!r} is not an integer") from None
    if not (-(1 << 63) <= n < (1 << 63)) or v.strip() != v or v.startswith("+"):
        raise StorageError(f"{what}: {v!r} is not an int64")
    return n


@dataclass
class NodeStorage:
    """utils.NodeStorage (pkg/utils/utils.go:510-513), parsed from the node annotation simon/node-local-storage."""
    vgs: Optional[List[list]]          # [name, capacity, requested] in annotation order; None: the JSON said null / nothing
    devices: Optional[List[dict]]      # kept as parsed: Bind rewrites them unchanged

    def to_json(self) -> str:
        """ffjson.Marshal(nodeStorage) as Bind writes it (open-local.go:242-246): compact, fields in struct order, int64 and
        bool fields with `,string` quoted."""
        def vg(v):
            return '{"name":%s,"capacity":"%d","requested":"%d"}' % (json.dumps(v[0], ensure_ascii=False), v[1], v[2])

        def dev(d):
            return ('{"name":%s,"device":%s,"capacity":"%d","mediaType":%s,"isAllocated":"%s"}' %
                    (json.dumps(d["name"], ensure_ascii=False), json.dumps(d["device"], ensure_ascii=False), d["capacity"],
                     json.dumps(d["mediaType"], ensure_ascii=False), "true" if d["isAllocated"] else "false"))
        vgs = "null" if self.vgs is None else "[" + ",".join(vg(v) for v in self.vgs) + "]"
        devs = "null" if self.devices is None else "[" + ",".join(dev(d) for d in self.devices) + "]"
        return '{"vgs":%s,"devices":%s}' % (vgs, devs)


def parse_node_storage(node: O.Obj, with_devices: bool = False) -> Optional[NodeStorage]:
    """GetNodeStorage / GetNodeCache (pkg/utils/utils.go:527-563).  None: no annotation.  A malformed annotation raises: the
    reference's Score parses the annotation of every feasible node for every pod and an error aborts the pod.
    with_devices: the node's SSD / HDD devices are placed, so duplicate device names (Bind marks the first entry of a name,
    open-local.go:232-238, which need not be the device the Filter chose) and more than MAX_DEVS of them are refused too."""
    ann = O.annotations_of(node)
    if O.ANNO_NODE_LOCAL_STORAGE not in ann:
        return None
    name = O.name_of(node)
    try:
        d = json.loads(ann[O.ANNO_NODE_LOCAL_STORAGE])
    except (ValueError, TypeError) as e:
        raise StorageError(f"node {name}: malformed {O.ANNO_NODE_LOCAL_STORAGE}: {e}") from None
    if d is None:
        return NodeStorage(None, None)
    if not isinstance(d, dict):
        raise StorageError(f"node {name}: {O.ANNO_NODE_LOCAL_STORAGE} is not an object")
    vgs = None
    if d.get("vgs") is not None:
        if not isinstance(d["vgs"], list):
            raise StorageError(f"node {name}: vgs is not a list")
        vgs = []
        for v in d["vgs"]:
            v = v or {}
            if not isinstance(v, dict) or not isinstance(v.get("name", ""), str):
                raise StorageError(f"node {name}: malformed VG entry")
            vgs.append([v.get("name", ""), _go_int_string(v.get("capacity", "0"), f"node {name} VG capacity"),
                        _go_int_string(v.get("requested", "0"), f"node {name} VG requested")])
    devices = None
    if d.get("devices") is not None:
        if not isinstance(d["devices"], list):
            raise StorageError(f"node {name}: devices is not a list")
        devices = []
        for v in d["devices"]:
            v = v or {}
            if not isinstance(v, dict):
                raise StorageError(f"node {name}: malformed device entry")
            alloc = v.get("isAllocated", "false")
            if alloc not in ("true", "false"):
                raise StorageError(f"node {name}: isAllocated must be \"true\" or \"false\"")
            devices.append(dict(name=str(v.get("name", "")), device=str(v.get("device", "")),
                                capacity=_go_int_string(v.get("capacity", "0"), f"node {name} device capacity"),
                                mediaType=str(v.get("mediaType", "")), isAllocated=alloc == "true"))
    # GetNodeCache keys VGs by name and devices by device: duplicates would collapse in the reference's maps
    names = [v[0] for v in vgs or []]
    if len(set(names)) != len(names):
        raise StorageError(f"node {name}: duplicate VG names")
    if "" in names:
        raise StorageError(f"node {name}: a VG named \"\"")
    devs = [x["device"] for x in devices or []]
    if len(set(devs)) != len(devs):
        raise StorageError(f"node {name}: duplicate device keys")
    if len(names) > MAX_VGS:
        raise StorageError(f"node {name}: more than {MAX_VGS} VGs")
    if with_devices:
        dnames = [x["name"] for x in devices or []]
        if len(set(dnames)) != len(dnames):
            raise StorageError(f"node {name}: duplicate device names")
        if sum(x["mediaType"] in MEDIA for x in devices or []) > MAX_DEVS:
            raise StorageError(f"node {name}: more than {MAX_DEVS} SSD / HDD devices")
    return NodeStorage(vgs, devices)


def storage_class_params(storage_classes: List[O.Obj]) -> Dict[str, Dict[str, str]]:
    """The StorageClass lister (OL/utils/common.go:301-342): name -> parameters; later objects of one name replace earlier ones."""
    out = {}
    for sc in storage_classes:
        out[O.name_of(sc)] = {str(k): str(v) for k, v in ((sc.get("parameters") or {}).items())}
    return out


@dataclass
class ClassVolumes:
    local: bool = False                                     # GetPodLocalPVCs returns some PVC: the plugin filters / scores
    dropped: int = 0                                        # device PVCs DividePVCAccordingToMediaType drops
    lvm: List[Tuple[int, str]] = field(default_factory=list)   # (size, vgName or "") in annotation order
    ssd: List[int] = field(default_factory=list)            # device PVC sizes, annotation order (devices=True only)
    hdd: List[int] = field(default_factory=list)


def pod_volumes(pod: O.Obj, sc_params: Dict[str, Dict[str, str]], devices: bool = False) -> ClassVolumes:
    """GetPodLocalPVCs (pkg/utils/utils.go:565-623) + DivideLVMPVCs / DividePVCAccordingToMediaType.  devices: SSD / HDD PVCs
    are kept for placement instead of refused."""
    ann = O.annotations_of(pod)
    cv = ClassVolumes()
    if O.ANNO_POD_LOCAL_STORAGE not in ann:
        return cv
    try:
        d = json.loads(ann[O.ANNO_POD_LOCAL_STORAGE])
        vols = [] if d is None else (d.get("volumes") or [])
        parsed = []
        for v in vols:
            v = v or {}
            parsed.append((str(v.get("kind", "")), _go_int_string(v.get("size", "0"), "size"), v.get("scName") or ""))
    except (ValueError, TypeError, AttributeError, StorageError):
        return cv                                            # GetPodStorage: an unmarshal error means no PVCs
    pname = f"{O.namespace_of(pod) or 'default'}/{O.name_of(pod)}"
    for kind, size, sc in parsed:
        if kind not in ("LVM", "HDD", "SSD"):
            continue
        cv.local = True
        params = sc_params.get(sc)
        if size <= 0:
            raise StorageError(f"pod {pname}: {kind} volume of size {size}: volumes of size 0 or less are not supported")
        if sc in LVM_SC:
            cv.lvm.append((size, (params or {}).get("vgName", "")))
        else:
            media = (params or {}).get("mediaType", "")
            if media in MEDIA:
                if not devices:
                    raise StorageError(f"pod {pname}: {media} device volume (StorageClass {sc}): exclusive Open-Local devices are "
                                       "not implemented by this engine without the devices opt-in")
                (cv.ssd if media == "ssd" else cv.hdd).append(size)
            else:
                cv.dropped += 1
    if len(cv.lvm) > MAX_VOLS:
        raise StorageError(f"pod {pname}: more than {MAX_VOLS} LVM volumes")
    if len(cv.ssd) + len(cv.hdd) > MAX_DEV_VOLS:
        raise StorageError(f"pod {pname}: more than {MAX_DEV_VOLS} SSD / HDD device volumes")
    return cv


def lvm_place(node_name: str, vgs: Optional[List[list]], lvm: List[Tuple[int, str]]):
    """ProcessLVMPVCPredicate (OL/scheduler/algorithm/algo/common.go:59-143) and the unit choice of ScoreLVMVolume / Binpack
    (:500-619) on one node's VGs ([name, capacity, requested], annotation order).
    Returns (error text or None, units [(vg index, size)], raw ScoreLVM (:660-692)).  Without LVM PVCs neither runs
    (open-local.go:76-81, ScoreLVMVolume :500-503): the node passes with score 0 whatever its VGs."""
    if not lvm:
        return None, [], 0
    vgs = vgs or []
    req = [v[2] for v in vgs]
    units = []
    idx = {v[0]: i for i, v in enumerate(vgs)}
    for size, vg in lvm:
        if not vg:
            continue
        i = idx.get(vg)
        if i is None:
            return f"not LVM named {vg}", [], 0                        # NotSuchVGError
        if vgs[i][1] - req[i] < size:
            return f"Insufficient LVM storage, requested {binary_si(size)}, used {binary_si(req[i])}, capacity {binary_si(vgs[i][1])}", [], 0
        req[i] += size
        units.append((i, size))
    if not vgs:
        return f"not LVM on node {node_name}", [], 0                   # NoAvailableVGError
    for size, vg in lvm:
        if vg:
            continue
        # the slice holds len(map) zero-valued VGs ahead of the real ones (make(len) + append), stably sorted by free size
        order = sorted([(0, -1)] * len(vgs) + [(vgs[i][1] - req[i], i) for i in range(len(vgs))], key=lambda t: t[0])
        pick = next((i for fr, i in order if i >= 0 and fr >= size), None)
        if pick is None:
            last = order[-1][1]
            used, cap = (req[last], vgs[last][1]) if last >= 0 else (0, 0)
            return f"Insufficient LVM storage, requested {binary_si(size)}, used {binary_si(used)}, capacity {binary_si(cap)}", [], 0
        req[pick] += size
        units.append((pick, size))
    used = {}
    for i, size in units:
        used[i] = used.get(i, 0) + size
    if not used:
        return None, units, 0
    sf = 0.0
    for i in sorted(used):
        sf += float(used[i]) / float(vgs[i][1])
    x = sf / float(len(used)) * 10.0
    return None, units, int(x)


def _insufficient_device(requested: int, available: int, capacity: int) -> str:
    # InsufficientExclusiveResourceError (OL/scheduler/errors/predicate.go:175-204), resource type "Device"
    return (f"Insufficient Device storage, requested {binary_si(requested)}, available {binary_si(available)}, "
            f"capacity {binary_si(capacity)}")


def device_place(node_name: str, devices: Optional[List[dict]], ssd: List[int], hdd: List[int]):
    """ProcessDevicePVC (OL/scheduler/algorithm/algo/common.go:394-448) with CheckExclusiveResourceMeetsPVCSize (:290-350), and
    ScoreDevice (:753-762), on one node's devices (annotation order, with the current isAllocated) for the SSD and HDD PVC sizes
    of a pod.  node_name is not part of any message; it keeps the signature of lvm_place.
    Returns (error text or None, annotation indices of the chosen devices, raw ScoreDevice).  The units are the SSD ones, then
    the HDD ones, each in ascending PVC size; without SSD / HDD PVCs the node passes with score 0 (ScoreDeviceVolume, :731-733;
    raw_score applies the all-dropped case)."""
    devices = devices or []
    total = len(devices)            # len(nodeCache.Devices): every device, allocated or not, of any media type
    free = {m: sorted((i for i, d in enumerate(devices) if d["mediaType"] == m and not d["isAllocated"]),
                      key=lambda i: devices[i]["capacity"]) for m in MEDIA}       # stable: ties in annotation order
    units = []
    for media, pvcs in zip(MEDIA, (ssd, hdd)):
        fr = free[media]
        if len(fr) < len(pvcs):
            # the HDD branch reports the SSD counts (common.go:430-435)
            return _insufficient_device(len(ssd), len(free["ssd"]), total), [], 0
        pvcs = sorted(pvcs)
        k = 0
        for j, i in enumerate(fr):
            if k == len(pvcs):
                break
            cap = devices[i]["capacity"]
            if cap < pvcs[k]:
                if j == len(fr) - 1:
                    return _insufficient_device(len(pvcs), len(fr), total), [], 0
                continue
            units.append((i, pvcs[k], cap))
            k += 1
        # devices that run out after a match leave the remaining PVCs without a unit, and the node passes (:312-349)
    if not units:
        return None, [], 0
    sf = 0.0
    for _i, req, cap in units:
        sf += float(req) / float(cap)
    return None, [i for i, _r, _c in units], int(sf / float(len(units)) * 10.0)


@dataclass
class StorageTables:
    """The simon_storage (and with devices=True simon_devices) columns plus what the host needs to turn engine results back into
    objects."""
    n_vgs: int
    node_n_vg: np.ndarray          # [N] int32
    vg_capacity: np.ndarray        # [V][N] int64
    vg_requested: np.ndarray       # [V][N] int64
    vg_name: np.ndarray            # [V][N] int32
    class_local: np.ndarray        # [C] uint8
    vol_off: np.ndarray            # [C+1] uint32
    vol_size: np.ndarray           # int64
    vol_vg: np.ndarray             # int32
    node_storage: List[Optional[NodeStorage]]     # per node (snapshot order)
    class_volumes: List[ClassVolumes]
    # SSD / HDD devices (devices=True): per node the slots 0 .. n_ssd-1 hold its SSDs, the next n_hdd its HDDs, each ascending by
    # capacity with ties in annotation order; devices of other media types have no slot
    devices: bool = False
    n_dev_slots: int = 0           # D <= MAX_DEVS
    node_n_ssd: Optional[np.ndarray] = None      # [N] uint8
    node_n_hdd: Optional[np.ndarray] = None      # [N] uint8
    dev_capacity: Optional[np.ndarray] = None    # [D][N] int64
    dev_index: Optional[np.ndarray] = None       # [D][N] int32 index into the annotation's "devices" list, -1: no device
    dev_alloc: Optional[np.ndarray] = None       # [N] uint32 bit s: slot s isAllocated
    ssd_off: Optional[np.ndarray] = None         # [C+1] uint32 offsets into ssd_size
    ssd_size: Optional[np.ndarray] = None        # int64, ascending per class
    hdd_off: Optional[np.ndarray] = None         # [C+1] uint32 offsets into hdd_size
    hdd_size: Optional[np.ndarray] = None        # int64, ascending per class

    def alloc_mask(self, g: int, devices: List[dict]) -> int:
        """Node g's slot mask of the allocated devices in `devices` (its annotation's list, possibly after binds)."""
        m = 0
        for s in range(int(self.node_n_ssd[g]) + int(self.node_n_hdd[g])):
            if devices[int(self.dev_index[s, g])]["isAllocated"]:
                m |= 1 << s
        return m


def compile_storage(snodes: List[O.Obj], class_pods: List[O.Obj], storage_classes: List[O.Obj],
                    devices: bool = False) -> StorageTables:
    """Columns of simon_storage for nodes in snapshot order and one representative pod per class; devices: also those of
    simon_devices, and SSD / HDD PVCs are placed instead of refused."""
    N, C = len(snodes), len(class_pods)
    ns = [parse_node_storage(n, devices) for n in snodes]
    V = max([len(s.vgs or []) for s in ns if s is not None] + [0])
    names: Dict[str, int] = {}
    node_n_vg = np.full(N, -1, np.int32)
    cap = np.zeros((V, N), np.int64)
    req = np.zeros((V, N), np.int64)
    nid = np.zeros((V, N), np.int32)
    for g, s in enumerate(ns):
        if s is None:
            continue
        node_n_vg[g] = len(s.vgs or [])
        for v, (nm, c, r) in enumerate(s.vgs or []):
            cap[v, g], req[v, g] = c, r
            nid[v, g] = names.setdefault(nm, len(names))
    params = storage_class_params(storage_classes)
    cvs = [pod_volumes(p, params, devices) for p in class_pods]
    class_local = np.array([1 if cv.local else 0 for cv in cvs], np.uint8)
    off, size, vgid = [0], [], []
    for cv in cvs:
        for sz, vg in cv.lvm:
            size.append(sz)
            # a vgName no node carries gets an id of its own: it matches no VG (NotSuchVGError everywhere)
            vgid.append(names.setdefault(vg, len(names)) if vg else -1)
        off.append(len(size))
    st = StorageTables(V, node_n_vg, cap, req, nid, class_local, np.array(off, np.uint32), np.array(size, np.int64),
                       np.array(vgid, np.int32), ns, cvs)
    if devices:
        _compile_devices(st)
    return st


def _compile_devices(st: StorageTables) -> None:
    N = len(st.node_storage)
    slots = []
    for s in st.node_storage:
        devs = (s.devices if s is not None else None) or []
        slots.append([sorted((i for i, d in enumerate(devs) if d["mediaType"] == m), key=lambda i: devs[i]["capacity"])
                      for m in MEDIA])
    D = max([len(a) + len(b) for a, b in slots] + [0])
    st.devices, st.n_dev_slots = True, D
    st.node_n_ssd = np.array([len(a) for a, _b in slots], np.uint8).reshape(N)
    st.node_n_hdd = np.array([len(b) for _a, b in slots], np.uint8).reshape(N)
    st.dev_capacity = np.zeros((D, N), np.int64)
    st.dev_index = np.full((D, N), -1, np.int32)
    st.dev_alloc = np.zeros(N, np.uint32)
    for g, (a, b) in enumerate(slots):
        devs = st.node_storage[g].devices if a or b else []
        for k, i in enumerate(a + b):
            st.dev_capacity[k, g], st.dev_index[k, g] = devs[i]["capacity"], i
        if a or b:
            st.dev_alloc[g] = st.alloc_mask(g, devs)
    for media in MEDIA:
        off, size = [0], []
        for cv in st.class_volumes:
            size += sorted(getattr(cv, media))
            off.append(len(size))
        setattr(st, media + "_off", np.array(off, np.uint32))
        setattr(st, media + "_size", np.array(size, np.int64))


def normalize_scores(raw: List[int]) -> List[int]:
    """NormalizeScore (open-local.go:146-171): min-max onto 0..100 (MinNodeScore 0, MaxNodeScore 100), from highest = -MaxInt64,
    lowest = MaxInt64; a zero range gives 0 everywhere.  Go int64 arithmetic (the differences here are small)."""
    hi, lo = -((1 << 63) - 1), (1 << 63) - 1
    for s in raw:
        hi, lo = max(hi, s), min(lo, s)
    rng = hi - lo
    return [0 if rng == 0 else (s - lo) * 100 // rng for s in raw]


def raw_score(cv: ClassVolumes, local_score: int) -> int:
    """Score (open-local.go:94-138) = ScoreLVMVolume + ScoreDeviceVolume; local_score: ScoreLVM + ScoreDevice of the placed
    units.  A class with device PVCs of which none is SSD or HDD (all dropped) has ScoreDevice of no units: int(NaN) = MinInt64
    on amd64 (common.go:753-762); it is the same on every node.  Any SSD or HDD PVC gives at least one unit on a node that passes."""
    return local_score + (INT64_MIN if cv.dropped and not cv.ssd and not cv.hdd else 0)


class StorageReplay:
    """Bind's effect on the node annotations, replayed in placement order from the engine's placements: the VG and device each
    PVC took depend only on the node's state and the class's volumes, so the host restates them without a device round trip."""

    def __init__(self, st: StorageTables, node_names: List[str]):
        self.st = st
        self.names = node_names
        self.vgs = [None if s is None or s.vgs is None else [list(v) for v in s.vgs] for s in st.node_storage]
        self.devs = [None if s is None or s.devices is None else [dict(d) for d in s.devices] for s in st.node_storage]
        self.touched = set()

    def place(self, cls: int, g: int):
        """(error text or None, LVM units, chosen device indices, raw score without the all-dropped offset) of a pod of class
        cls on node g's current state: the LVM part first, then the devices (open-local.go:75-89)."""
        cv = self.st.class_volumes[cls]
        err, units, s1 = lvm_place(self.names[g], self.vgs[g], cv.lvm)
        if err is not None:
            return err, [], [], 0
        err, chosen, s2 = device_place(self.names[g], self.devs[g], cv.ssd, cv.hdd)
        if err is not None:
            return err, [], [], 0
        return None, units, chosen, s1 + s2

    def bind(self, cls: int, g: int):
        cv = self.st.class_volumes[cls]
        if not cv.local or self.st.node_storage[g] is None:
            return
        err, units, chosen, _ = self.place(cls, g)
        assert err is None, f"engine placed a pod of class {cls} on node {self.names[g]} that Open-Local rejects: {err}"
        for i, size in units:
            self.vgs[g][i][2] += size
        for i in chosen:        # device names are unique per node (parse_node_storage): the entry of the name is the chosen one
            self.devs[g][i]["isAllocated"] = True
        self.touched.add(g)

    def reason(self, cls: int, g: int) -> Optional[str]:
        """The Filter's status message of node g for a pod of class cls (None: Unschedulable without a reason)."""
        if self.st.node_storage[g] is None:
            return None
        return self.place(cls, g)[0]

    def requested(self) -> np.ndarray:
        V, N = self.st.n_vgs, len(self.names)
        out = np.array(self.st.vg_requested, copy=True).reshape(V, N)
        for g, vs in enumerate(self.vgs):
            for v, x in enumerate(vs or []):
                out[v, g] = x[2]
        return out

    def alloc_masks(self) -> np.ndarray:
        """[N] slot masks of the allocated devices (the simon_devices state)."""
        out = np.array(self.st.dev_alloc, copy=True)
        for g in self.touched:
            if self.devs[g]:
                out[g] = self.st.alloc_mask(g, self.devs[g])
        return out

    def annotation(self, g: int) -> Optional[str]:
        """The node annotation after the replayed binds; None where no Bind touched the node (the original text stays)."""
        if g not in self.touched:
            return None
        return NodeStorage(self.vgs[g], self.devs[g]).to_json()
