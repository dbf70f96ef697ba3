"""Drives a running sdwui-API worker server with the UNMODIFIED reference `Worker` class (/root/reference), in its own
process because the reference's module names (`scripts.spartan.*`) are the same as this repo's.

    REFERENCE_DIR=<reference checkout> python tests/ref_rest_probe.py <port>   -> one JSON line on stdout

tests/golden/gen_ref_rest_golden.py runs it once against the REST server and stores what it saw (the HTTP exchanges
and the values the reference Worker parsed out of them) in tests/golden/ref_rest_golden.json, which
tests/test_rest_worker_cpu.py replays.
"""
import base64
import io
import json
import logging.handlers
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("REFERENCE_DIR", "/root/reference")
tmp = tempfile.mkdtemp(prefix="refprobe_")
os.environ["HOSTSTUB_CONFIG_DIR"] = tmp
sys.path[:0] = [os.path.join(HERE, "hoststub"), REF]

import pydantic.v1  # noqa: E402

sys.modules["pydantic"] = pydantic.v1
_Orig = logging.handlers.RotatingFileHandler


class _Redirected(_Orig):
    def __init__(self, filename, *a, **k):
        super().__init__(os.path.join(tmp, os.path.basename(str(filename))), *a, **k)


logging.handlers.RotatingFileHandler = _Redirected

from scripts.spartan import pmodels, shared, worker  # noqa: E402  (the reference's)

logging.getLogger("distributed").setLevel(logging.CRITICAL + 1)
shared.benchmark_payload = pmodels.Benchmark_Payload()  # what World.load_config() installs (world.py:672-676)


EXCHANGES = []  # every HTTP exchange the reference Worker makes: (method, path, JSON body) -> (status, JSON reply)


def _recording(orig):
    from urllib.parse import urlsplit

    def request(self, method, url, *a, **k):
        r = orig(self, method, url, *a, **k)
        try:
            reply = r.json()
        except ValueError:
            reply = None
        EXCHANGES.append({"method": method.upper(), "path": urlsplit(url).path, "json": k.get("json"),
                          "status": r.status_code, "reply": reply})
        return r
    return request


def main():
    port = int(sys.argv[1])
    import requests
    requests.Session.request = _recording(requests.Session.request)
    w = worker.Worker(address="127.0.0.1", port=port, label="b200box", verify_remotes=False, avg_ipm=600.0)
    out = {"reference_file": worker.__file__, "reachable": bool(w.reachable())}
    w.benchmarked = True
    payload = {"prompt": "a probe", "negative_prompt": "", "seed": 31, "subseed": 7, "subseed_strength": 0, "batch_size": 2,
               "n_iter": 1, "steps": 4, "width": 64, "height": 64, "sampler_name": "DDIM", "cfg_scale": 7.0,
               "s_tmax": float("inf"), "alwayson_scripts": {}}
    w.request(dict(payload), {"sd_model_checkpoint": "m.safetensors", "sd_vae": None}, True)
    r = w.response
    out["state"] = w.state.name
    out["n_images"] = len(r["images"])
    info = json.loads(r["info"])
    out["all_seeds"] = info["all_seeds"]
    out["all_subseeds"] = info["all_subseeds"]
    from PIL import Image
    import hashlib
    import numpy as np
    out["image_sha1"] = [hashlib.sha1(np.asarray(Image.open(io.BytesIO(base64.b64decode(s)))).tobytes()).hexdigest()
                         for s in r["images"]]
    out["loaded_model"] = w.loaded_model
    out["models"] = w.available_models()
    out["exchanges"] = EXCHANGES
    print(json.dumps(out))


if __name__ == "__main__":
    main()
