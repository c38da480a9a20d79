"""N-pipelines-on-N-GPUs plumbing (SURVEY §8e): one process per GPU, independent streams, no
collective on the data path.  torch.distributed is used only to line the ranks up and to take the
max over ranks of per-rank timings / sum of per-rank frame counts."""
import os


def rank_info():
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")),
            int(os.environ.get("LOCAL_RANK", "0")))


def init(backend=None, device=None):
    """returns the torch.distributed module when WORLD_SIZE > 1, else None"""
    rank, world, local = rank_info()
    if world <= 1:
        return None
    import torch
    import torch.distributed as dist
    if backend is None:
        backend = "nccl" if torch.cuda.is_available() else "gloo"
    kw = {}
    if backend == "nccl" and device is not None:
        kw["device_id"] = device
    dist.init_process_group(backend, **kw)
    return dist


def reduce_max(dist, values, device="cpu"):
    """max over ranks of a list of floats (device timings are reported as the slowest rank)"""
    import torch
    t = torch.tensor(list(values), dtype=torch.float64, device=device)
    if dist is not None:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return [float(x) for x in t]


def reduce_sum(dist, values, device="cpu"):
    import torch
    t = torch.tensor(list(values), dtype=torch.float64, device=device)
    if dist is not None:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return [float(x) for x in t]


def stream_seed(rank, frame):
    """distinct synthetic content per (pipeline, frame): each rank is its own video stream"""
    return 1000 * rank + frame


def whole_job_throughput(units_per_rank, world, seconds_max):
    """weak scaling: every rank processes the same number of units; the job's rate is all units
    over the slowest rank's time"""
    return units_per_rank * world / seconds_max


def gpu_numa_cpus(local_gpu):
    """(numa node, cpu list) the GPU hangs off, from sysfs (nvidia-smi topo prints the same affinity); (None, []) if unknown"""
    try:
        import pynvml as nv
        nv.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "")
        idx = local_gpu
        ids = [v for v in vis.split(",") if v.strip()]
        if ids and local_gpu < len(ids) and ids[local_gpu].strip().isdigit():
            idx = int(ids[local_gpu])
        pci = nv.nvmlDeviceGetPciInfo(nv.nvmlDeviceGetHandleByIndex(idx)).busId
        pci = pci.decode() if isinstance(pci, bytes) else pci
        pci = pci.lower()
        if len(pci.split(":")[0]) == 8:          # NVML prints an 8-digit domain, sysfs a 4-digit one
            pci = pci[4:]
        base = "/sys/bus/pci/devices/" + pci
        node = int(open(base + "/numa_node").read())
        cpus = _parse_cpulist(open(base + "/local_cpulist").read())
        return (node if node >= 0 else None), cpus
    except Exception:
        return None, []


def _parse_cpulist(text):
    out = []
    for part in text.strip().split(","):
        if not part:
            continue
        a, _, b = part.partition("-")
        out.extend(range(int(a), int(b or a) + 1))
    return out


def bind_to_gpu_numa(local_gpu):
    """Pin this process (one pipeline per GPU) to the cores next to its GPU, BEFORE any staging memory is allocated or
    touched: one pipeline per GPU on a two-socket host otherwise pushes half of the H2D / D2H bytes across the socket
    interconnect.  Returns what it did, for the bench line."""
    node, cpus = gpu_numa_cpus(local_gpu)
    if not cpus:
        return {"numa_node": node, "bound": False}
    try:
        os.sched_setaffinity(0, cpus)
        return {"numa_node": node, "bound": True, "cpus": len(cpus)}
    except Exception as e:          # cgroup cpuset narrower than the GPU's local list
        try:
            allowed = sorted(set(cpus) & os.sched_getaffinity(0))
            if allowed:
                os.sched_setaffinity(0, allowed)
                return {"numa_node": node, "bound": True, "cpus": len(allowed)}
        except Exception:
            pass
        return {"numa_node": node, "bound": False, "error": str(e)}
