"""How many CPUs may this process really use (affinity mask and cgroup quota, not `os.cpu_count()`)."""
import os


def usable_cpus() -> int:
    """CPUs this process may actually USE: the smaller of the affinity mask and the cgroup CPU quota.  In a container
    `os.cpu_count()` can report every host core while the quota (`cpu.max`, e.g. "1600000 100000") allows 16 - sizing a
    decode pool by the former oversubscribes it and loses throughput."""
    try:
        n = len(os.sched_getaffinity(0))
    except (AttributeError, OSError):
        n = os.cpu_count() or 1
    try:
        with open("/sys/fs/cgroup/cpu.max") as f:           # cgroup v2
            quota, period = f.read().split()[:2]
        if quota != "max":
            n = min(n, max(1, int(int(quota) / int(period) + 0.5)))
    except (OSError, ValueError):
        try:                                                  # cgroup v1
            with open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us") as f:
                quota = int(f.read())
            with open("/sys/fs/cgroup/cpu/cpu.cfs_period_us") as f:
                period = int(f.read())
            if quota > 0 and period > 0:
                n = min(n, max(1, int(quota / period + 0.5)))
        except (OSError, ValueError):
            pass
    return max(1, n)
