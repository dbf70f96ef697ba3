"""Records tests/golden/ref_rest_golden.json: the UNMODIFIED reference `Worker` (scripts/spartan/worker.py of the
reference checkout named by REFERENCE_DIR) driving this repo's REST worker server (server/sdapi.py, deterministic engine
double of tests/test_rest_worker_cpu.py) over real HTTP.  Stored: every request it sent (method, path, JSON body), every
reply (status, JSON; base64 PNG images replaced by the SHA-1 of their decoded pixels) and the values it parsed out of them.
tests/test_rest_worker_cpu.py replays the requests against the server and compares, so the reference is needed only here.

    REFERENCE_DIR=<reference checkout> python tests/golden/gen_ref_rest_golden.py
"""
import json
import os
import subprocess
import sys
import threading
import time

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
sys.path[:0] = [TESTS, ROOT, os.path.join(ROOT, "stable-diffusion-webui-distributed_b200")]

from test_rest_worker_cpu import EngineDouble, _free_port, strip_images  # noqa: E402


def main():
    import uvicorn
    from server.sdapi import create_app
    eng = EngineDouble()
    port = _free_port()
    srv = uvicorn.Server(uvicorn.Config(create_app(lambda device: eng, [0]), host="127.0.0.1", port=port, log_level="error"))
    t = threading.Thread(target=srv.run, daemon=True)
    t.start()
    while not srv.started:
        time.sleep(0.05)
    p = subprocess.run([sys.executable, os.path.join(TESTS, "ref_rest_probe.py"), str(port)], capture_output=True, text=True,
                       timeout=120, check=True)
    srv.should_exit = True
    t.join(timeout=5)
    out = json.loads(p.stdout.strip().splitlines()[-1])
    del out["reference_file"]
    for ex in out["exchanges"]:
        ex["reply"] = strip_images(ex["reply"])
    with open(os.path.join(HERE, "ref_rest_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
