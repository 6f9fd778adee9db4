"""``python -m torchft_b200.doctor [--lighthouse http://host:29510]`` — is this box ready for the native data plane?

Prints one line per check (OK / WARN / FAIL) and exits non-zero when something REQUIRED for the requested mode is
missing: native extensions built and importable, CUDA devices and their compute capability (sm_90 expected), peer
access between every GPU pair (the peer-memory collectives need it), NVSwitch multicast support (NVLS kernels, VMM
mode), shared-memory / file-descriptor limits that the fd-passing path needs, and — optionally — whether a Lighthouse
answers. Every probe is independent and never raises.
"""

from __future__ import annotations

import argparse
import os
import resource
import sys
from datetime import timedelta
from typing import Callable, List, Tuple

Check = Tuple[str, str, str]  # (level, name, detail)


def _probe(name: str, fn: Callable[[], Tuple[str, str]], out: List[Check]) -> None:
    try:
        level, detail = fn()
    except Exception as e:  # noqa: BLE001 - a doctor must survive its patients
        level, detail = "FAIL", f"{type(e).__name__}: {e}"
    out.append((level, name, detail))


def run(lighthouse: str = "", require_gpu: bool = False) -> List[Check]:
    out: List[Check] = []

    def ext_control() -> Tuple[str, str]:
        from torchft_b200 import _C

        return "OK", f"control plane module {_C.__file__}"

    def ext_kernels() -> Tuple[str, str]:
        import glob

        so = glob.glob(os.path.join(os.path.dirname(__file__), "_K*.so"))
        if not so:
            return "FAIL", "kernel module not built: run `python -m torchft_b200._build`"
        return "OK", f"kernel module {so[0]} ({os.path.getsize(so[0]) >> 20} MiB)"

    def selftest() -> Tuple[str, str]:
        exe = os.path.join(os.path.dirname(os.path.dirname(__file__)), "bin", "torchft_b200_selftest")
        return ("OK", exe) if os.path.exists(exe) else ("WARN", "native selftest binary not built (optional)")

    _probe("extension _C", ext_control, out)
    _probe("extension _K", ext_kernels, out)
    _probe("native selftest", selftest, out)

    def fds() -> Tuple[str, str]:
        soft, hard = resource.getrlimit(resource.RLIMIT_NOFILE)
        return ("OK" if soft >= 4096 else "WARN"), f"RLIMIT_NOFILE soft={soft} hard={hard} (thread-per-connection servers + fd passing)"

    _probe("file descriptors", fds, out)

    import torch

    ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if ngpu == 0:
        out.append(("FAIL" if require_gpu else "WARN", "cuda", "no CUDA device visible: only the CPU (Gloo) data plane is usable here"))
    else:
        def devices() -> Tuple[str, str]:
            caps = {torch.cuda.get_device_capability(i) for i in range(ngpu)}
            names = {torch.cuda.get_device_name(i) for i in range(ngpu)}
            ok = caps == {(9, 0)}
            return ("OK" if ok else "FAIL"), f"{ngpu} x {', '.join(sorted(names))}, compute capability {sorted(caps)} (kernels are built for sm_90a only)"

        def peers() -> Tuple[str, str]:
            bad = [(i, j) for i in range(ngpu) for j in range(ngpu) if i != j and not torch.cuda.can_device_access_peer(i, j)]
            return ("OK", f"peer access between all {ngpu * (ngpu - 1)} ordered GPU pairs") if not bad else ("FAIL", f"no peer access for pairs {bad[:6]}")

        def multicast() -> Tuple[str, str]:
            from torchft_b200.ops import _native

            K = _native.load()
            ok = True
            for i in range(ngpu):
                with torch.cuda.device(i):  # the probe asks about the CURRENT device
                    ok = ok and bool(K.multicast_supported())
            return ("OK", "NVSwitch multicast supported on every device (TORCHFT_B200_SYMM=vmm enables the NVLS kernel)") if ok else (
                "WARN", "multicast not supported: VMM mode works, the NVLS kernel is unavailable")

        def memory() -> Tuple[str, str]:
            free, total = torch.cuda.mem_get_info(0)
            return "OK", f"GPU0 memory {free / 2**30:.0f} / {total / 2**30:.0f} GiB free (Llama-3-8B full replica needs ~131 GiB)"

        _probe("devices", devices, out)
        _probe("peer access", peers, out)
        _probe("multicast", multicast, out)
        _probe("memory", memory, out)

    if lighthouse:
        def lh() -> Tuple[str, str]:
            from torchft_b200.coordination import wait_for_lighthouse

            st = wait_for_lighthouse(lighthouse, timedelta(seconds=5))
            n = len((st.get("prev_quorum") or {}).get("participants", []))
            return "OK", f"lighthouse answers: quorum_id={st['quorum_id']}, {n} replicas in the last quorum, min_replicas={st['min_replicas']}"

        _probe("lighthouse", lh, out)
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lighthouse", default=os.environ.get("TORCHFT_LIGHTHOUSE", ""))
    ap.add_argument("--require-gpu", action="store_true")
    a = ap.parse_args()
    checks = run(a.lighthouse, a.require_gpu)
    for level, name, detail in checks:
        print(f"[{level:4s}] {name:18s} {detail}")
    sys.exit(1 if any(level == "FAIL" for level, _, _ in checks) else 0)


if __name__ == "__main__":
    main()
