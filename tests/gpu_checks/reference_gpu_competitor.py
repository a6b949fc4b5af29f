"""Same-box GPU competitor (SURVEY.md §8d): the reference's own CUDA/cuDNN backend against the reference search on OUR backend,
both through the reference's `katago benchmark` command (multi-threaded search of a few fixed 19x19 positions).

    gpurun --timeout 900 -- 'python tests/gpu_checks/reference_gpu_competitor.py > gpurun_out/competitor.json'

Needs oracle/_ref/katago_cuda (oracle/Makefile.cuda) and oracle/_ref/katago_b200 (oracle/Makefile.drivers), both built where the
reference sources are and shipped with the snapshot.  Random-weight b18c384nbt (no network for real nets): policies are near
uniform, trees wide and shallow - the same caveat as bench.py's.  Not a bench.py line: a measurement note."""
import json, os, re, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import modelgen

CFG = """logDir = {logdir}
logAllGTPCommunication = false
logSearchInfo = false
logToStderr = false
rules = tromp-taylor
numSearchThreads = 256
nnMaxBatchSize = 256
nnCacheSizePowerOfTwo = 20
nnMutexPoolSizePowerOfTwo = 16
nnRandomize = true
maxVisits = 600
{extra}
"""


def run(binary, model, cfg, threads, visits, timeout):
    cmd = [binary, "benchmark", "-model", model, "-config", cfg, "-v", str(visits), "-t", ",".join(map(str, threads)), "-n", "6"]
    try:
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout)
    except subprocess.TimeoutExpired:
        return {"error": "timeout"}
    out = p.stdout + p.stderr
    best = {}
    for m in re.finditer(r"numSearchThreads = +(\d+): +(\d+) / (\d+) positions, visits/s = ([\d.]+)", out):
        if m.group(2) == m.group(3):
            best[int(m.group(1))] = float(m.group(4))
    res = {"returncode": p.returncode, "visits_per_sec_by_threads": best}
    if not best:
        res["tail"] = out[-1500:]
    return res


def main():
    model_name = sys.argv[1] if len(sys.argv) > 1 else "b18c384nbt"
    d = tempfile.mkdtemp(prefix="kgb_competitor_")
    model = modelgen.write_model(os.path.join(d, model_name + ".bin.gz"), model_name, seed=0)
    out = {"model": model_name, "visits": 600, "positions": 6}
    for name, binary, extra in (("reference_cuda_backend_fp16", "katago_cuda", "cudaUseFP16 = true\ncudaUseNHWC = true"),
                                ("reference_search_on_b200_backend", "katago_b200", "")):
        path = os.path.join(ROOT, "oracle", "_ref", binary)
        if not os.path.exists(path):
            out[name] = {"error": "binary not built"}
            continue
        cfg = os.path.join(d, binary + ".cfg")
        open(cfg, "w").write(CFG.format(logdir=os.path.join(d, "logs_" + binary), extra=extra))
        out[name] = run(path, model, cfg, [64, 128, 256, 512], 600, 400)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
