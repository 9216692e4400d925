"""Batch sharding across the GPUs of one box (SURVEY.md section 8e).

The LQR step is independent per problem, so a rank only needs its own dense shard of every
``[T,B,...]`` tensor (dim 1) and of ``x_init`` (dim 0); there is NO collective on the solve path.
Collectives (NCCL on GPUs, gloo in the CPU tests) are used only to present gathered outputs and for
the optional global early-stop of the outer loop (reference mpc/mpc.py:299: ``max(full_du_norm) < eps``
is a batch-wide test)."""
import torch
import torch.distributed as dist


def shard_range(n_batch, rank, world):
    """Contiguous, balanced [lo, hi) of the batch owned by `rank`."""
    base, rem = divmod(n_batch, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_problem(rank, world, x_init, C, c, F, f=None, **per_time_batch):
    """Dense per-rank shards (time-major layout makes a dim-1 slice strided, hence .contiguous())."""
    lo, hi = shard_range(C.shape[1], rank, world)
    out = dict(x_init=x_init[lo:hi].contiguous(), C=C[:, lo:hi].contiguous(), c=c[:, lo:hi].contiguous(),
               F=F[:, lo:hi].contiguous(), f=None if f is None or f.nelement() == 0 else f[:, lo:hi].contiguous())
    for k, v in per_time_batch.items():
        out[k] = v[:, lo:hi].contiguous() if torch.is_tensor(v) else v
    return out


def gather_batch(t, dim, n_batch, group=None):
    """all_gather of a per-rank shard along `dim` (uneven shards allowed)."""
    world = dist.get_world_size(group)
    if world == 1:
        return t
    sizes = [hi - lo for lo, hi in (shard_range(n_batch, r, world) for r in range(world))]
    longest = max(sizes)
    t = t.contiguous()
    if t.shape[dim] < longest:                      # equal-size buffers: pad the short shards
        pad_shape = list(t.shape)
        pad_shape[dim] = longest - t.shape[dim]
        t = torch.cat((t, t.new_zeros(pad_shape)), dim)
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t, group=group)
    return torch.cat([p.narrow(dim, 0, sz) for p, sz in zip(parts, sizes)], dim)


def global_max(value, group=None):
    """max over ranks of a 0-d/1-element tensor (global early-stop test of the outer loop)."""
    v = value.detach().reshape(1).clone()
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(v, op=dist.ReduceOp.MAX, group=group)
    return v[0]


# ----------------------------------------------------------------------------------------------
# host staging buffers: pinned memory on the GPU's own NUMA node
# ----------------------------------------------------------------------------------------------
def gpu_local_cpus(device):
    """CPU ids the driver reports as local to `device` (NVML cpu affinity), restricted to this process'
    allowed set; None when NVML / the PCI id is unavailable.  One process per GPU, so this is also the right
    set to run the rank's host threads on."""
    import os
    try:
        import pynvml
        pr = torch.cuda.get_device_properties(device)
        bus = "%08x:%02x:%02x.0" % (pr.pci_domain_id, pr.pci_bus_id, pr.pci_device_id)
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByPciBusId(bus.encode())
        words = pynvml.nvmlDeviceGetCpuAffinity(h, (os.cpu_count() + 63) // 64)
        cpus = {64 * i + b for i, w in enumerate(words) for b in range(64) if (int(w) >> b) & 1}
        cpus &= os.sched_getaffinity(0)
        return cpus or None
    except Exception:                               # noqa: BLE001 - best effort: any failure means "do not pin"
        return None


class numa_local:
    """``with numa_local(device): buf = t.pin_memory()`` - allocate (first-touch) host staging buffers while the
    thread runs on the GPU's local cores, so the pinned pages live on the socket the GPU hangs off.  A copy from
    the far socket crosses the inter-socket link, which is slower than the GPU's own PCIe link."""

    def __init__(self, device):
        self.cpus = gpu_local_cpus(device)
        self.saved = None

    def __enter__(self):
        import os
        if self.cpus:
            try:
                self.saved = os.sched_getaffinity(0)
                os.sched_setaffinity(0, self.cpus)
            except OSError:
                self.saved = None
        return self

    def __exit__(self, *exc):
        import os
        if self.saved is not None:
            os.sched_setaffinity(0, self.saved)


def pin_local(t, device):
    """Pinned host copy of `t` placed on `device`'s NUMA node (see numa_local)."""
    with numa_local(device):
        return t.cpu().pin_memory()
