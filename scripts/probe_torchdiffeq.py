"""Is a real torchdiffeq (or torchsde / the reference torchcde) importable on this machine?

VERDICT r01 item 1: the stepping arithmetic behind torchcde/solver.py:226-227 lives in torchdiffeq, which is
not vendored.  This probe records -- as evidence, not assumption -- whether the package exists on the box the
benchmarks run on.  If it does, the restated solvers (oracle/odeint_port.py, torchcde_b200/adaptive.py) are
diffed against it on a small seeded problem and the differences are printed; if not, the module search path and
the installed distributions are logged.  Output goes to stdout.
"""
import importlib.metadata
import importlib.util
import os
import platform
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    print("# torchdiffeq probe")
    print("host:", platform.node(), "| python", sys.version.split()[0], "| torch", torch.__version__, "| cuda available:",
          torch.cuda.is_available(), "|", torch.cuda.get_device_name(0) if torch.cuda.is_available() else "no GPU")
    found = {}
    for name in ("torchdiffeq", "torchsde", "torchcde", "signatory"):
        try:
            spec = importlib.util.find_spec(name)
        except (ImportError, ValueError) as exc:
            spec = None
            print("find_spec({!r}) raised {!r}".format(name, exc))
        found[name] = spec
        print("find_spec({!r}): {}".format(name, spec.origin if spec else None))
    from oracle import reference_loader
    print("reference tree present:", reference_loader.reference_available())
    print("baseline/_ref present:", os.path.isdir(os.path.join(ROOT, "baseline", "_ref")))
    dists = sorted({d.metadata["Name"] for d in importlib.metadata.distributions() if d.metadata["Name"]}, key=str.lower)
    hits = [d for d in dists if any(k in d.lower() for k in ("diffeq", "torchsde", "torchcde", "signatory"))]
    print("installed distributions: {} total; ODE-related: {}".format(len(dists), hits or "none"))
    wheel_dir = "/opt/wheelhouse"
    if os.path.isdir(wheel_dir):
        wheels = [w for w in os.listdir(wheel_dir) if any(k in w.lower() for k in ("diffeq", "torchsde", "torchcde"))]
        print("/opt/wheelhouse: {} files; ODE-related: {}".format(len(os.listdir(wheel_dir)), wheels or "none"))
    else:
        print("/opt/wheelhouse: absent")
    print("sys.path:", [p for p in sys.path if p])

    if found["torchdiffeq"] is None:
        print("RESULT: torchdiffeq ABSENT on this machine -> the stepping oracle (oracle/odeint_port.py) stays anchored on "
              "analytic solutions / convergence orders only (parity unpinned).")
        return 0

    import torchdiffeq
    from oracle import odeint_port
    print("torchdiffeq version:", getattr(torchdiffeq, "__version__", "?"))
    torch.manual_seed(0)
    a = torch.randn(6, 6, dtype=torch.float64) * 0.3

    def field(t, y):
        return torch.tanh(y @ a.T) * torch.cos(t) + 0.1 * y

    y0 = torch.randn(5, 6, dtype=torch.float64)
    worst = 0.0
    for method in ("euler", "midpoint", "rk4"):
        for step in (None, 0.25, 0.3):
            for ts in ([0.0, 1.0, 2.5], [0.0, 0.4, 0.7, 2.0], [2.0, 1.1, 0.0]):
                t = torch.tensor(ts, dtype=torch.float64)
                opts = {} if step is None else {"step_size": step}
                want = torchdiffeq.odeint(field, y0, t, method=method, options=opts)
                got = odeint_port.odeint(field, y0, t, method=method, options=opts)
                err = (want - got).abs().max().item()
                worst = max(worst, err)
                print("odeint {:8s} step={} t={}: max |port - torchdiffeq| = {:.3e}".format(method, step, ts, err))
    print("RESULT: torchdiffeq PRESENT; worst fixed-grid difference {:.3e}".format(worst))
    return 0


if __name__ == "__main__":
    sys.exit(main())
