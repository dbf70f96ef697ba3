"""sdwui-compatible REST worker backed by the H100 executor (SURVEY.md §8 row f1).

The reference reaches its workers only through nine sdwui API routes (SURVEY §2.2; all issued from
scripts/spartan/worker.py and world.py of the reference):

    POST /sdapi/v1/txt2img, /sdapi/v1/img2img   worker.py:432-435   the generation RPC
    GET  /sdapi/v1/memory                        worker.py:322-331, :608-611   VRAM query / reachability ping
    POST /sdapi/v1/options                       worker.py:665-668   checkpoint / VAE sync
    POST /sdapi/v1/interrupt                     worker.py:597
    POST /sdapi/v1/refresh-checkpoints, /refresh-loras   worker.py:580-581
    GET  /sdapi/v1/sd-models                     worker.py:629-632
    POST /sdapi/v1/server-restart                worker.py:698
    GET  /sdapi/v1/script-info                   world.py:750

This module serves exactly those, with the reply shapes the reference reads, on top of `LocalGPUWorker` — so an
UNMODIFIED reference master (or this repo's `Worker` with its HTTP transport) can list an H100 node in its
`distributed-config.json` like any other sdwui node.  One process serves the GPUs of one box: requests are dispatched to
the least-loaded device, one generation per device at a time (the executor replays CUDA graphs; the GIL is idle).

    python -m server.sdapi --port 7860 --devices 0,1,2,3        (from stable-diffusion-webui-distributed_b200/)

Images travel as base64 PNG (the API's wire format); the in-process fast lane (`response["tensors"]`) is not available
over HTTP.  Optional HTTP basic auth mirrors sdwui's `--api-auth user:password`.
"""
import argparse
import secrets
import threading
import time
from typing import Callable, List, Optional

from fastapi import Depends, FastAPI, HTTPException, Request
from fastapi.security import HTTPBasic, HTTPBasicCredentials

API = "/sdapi/v1"


class DevicePool:
    """one LocalGPUWorker per device; a request takes the device with the fewest requests in flight"""

    def __init__(self, engine_factory: Callable, devices: List[int]):
        from . import standalone_host
        standalone_host.install()  # no-op inside sdwui
        from scripts.spartan.local_worker import LocalGPUWorker
        self.workers = [LocalGPUWorker(d, engine_factory, label=f"gpu{d}", png_images=True) for d in devices]
        self.locks = [threading.Lock() for _ in devices]
        self.inflight = [0] * len(devices)
        self._mu = threading.Lock()

    def run(self, payload: dict) -> dict:
        with self._mu:
            i = min(range(len(self.workers)), key=lambda k: self.inflight[k])
            self.inflight[i] += 1
        try:
            with self.locks[i]:
                return self.workers[i]._generate(payload)
        finally:
            with self._mu:
                self.inflight[i] -= 1

    def interrupt(self):
        for w in self.workers:
            if w._engine is not None:
                w._engine.interrupted = True

    def restart(self):
        """drop every device's engine — after the generation it is serving, never under it"""
        for w, lock in zip(self.workers, self.locks):
            with lock:
                w.restart()


MAX_BATCH = 64      # images per call and device
MAX_SIDE = 2048     # pixels


def _jsonable_reply(rep: dict) -> dict:
    """the API reply: images / parameters / info only (the host-tensor fast lane stays in-process)"""
    return {"images": rep["images"], "parameters": rep["parameters"], "info": rep["info"]}


def create_app(engine_factory: Callable, devices: Optional[List[int]] = None, api_auth: Optional[str] = None,
               model_title: str = "b200sd-synthetic.safetensors [00000000]") -> FastAPI:
    app = FastAPI(title="b200sd sdwui-API worker")
    pool = DevicePool(engine_factory, devices if devices else [0])
    app.state.pool = pool
    app.state.options = {"sd_model_checkpoint": model_title, "sd_vae": None}
    app.state.started = time.time()
    security = HTTPBasic(auto_error=False)

    def auth(cred: Optional[HTTPBasicCredentials] = Depends(security)):
        if api_auth is None:
            return
        user, _, pw = api_auth.partition(":")
        if cred is None or not (secrets.compare_digest(cred.username, user) and secrets.compare_digest(cred.password, pw)):
            raise HTTPException(status_code=401, detail="Incorrect username or password",
                                headers={"WWW-Authenticate": "Basic"})

    async def _generate(request: Request, img2img: bool):
        payload = await request.json()
        if not isinstance(payload, dict):
            raise HTTPException(status_code=422, detail="payload must be a JSON object")
        payload.setdefault("batch_size", 1)
        payload.setdefault("n_iter", 1)
        payload.setdefault("steps", 20)
        payload.setdefault("width", 512)
        payload.setdefault("height", 512)
        # bound what one request may allocate: every distinct (batch, size) builds activation buffers and graphs
        try:
            bs, ni = int(payload["batch_size"]), int(payload["n_iter"])
            wd, ht, st = int(payload["width"]), int(payload["height"]), int(payload["steps"])
        except (TypeError, ValueError):
            raise HTTPException(status_code=422, detail="batch_size, n_iter, steps, width, height must be integers")
        if not (1 <= bs <= MAX_BATCH and 1 <= ni <= 64 and 1 <= st <= 150 and 64 <= wd <= MAX_SIDE and 64 <= ht <= MAX_SIDE
                and wd % 64 == 0 and ht % 64 == 0):
            raise HTTPException(status_code=422, detail=f"out of range: batch_size 1..{MAX_BATCH}, n_iter 1..64, steps 1..150, "
                                                         f"width/height multiples of 64 in 64..{MAX_SIDE}")
        if img2img and not payload.get("init_images"):
            raise HTTPException(status_code=404, detail="Init image not found")
        if not img2img:
            payload.pop("init_images", None)
        try:
            import anyio
            rep = await anyio.to_thread.run_sync(pool.run, payload)
        except NotImplementedError as e:
            raise HTTPException(status_code=422, detail=str(e))
        except Exception as e:  # the reference treats any non-200 as a failed job (worker.py:469-473)
            raise HTTPException(status_code=500, detail=f"{type(e).__name__}: {e}")
        return _jsonable_reply(rep)

    @app.post(f"{API}/txt2img", dependencies=[Depends(auth)])
    async def txt2img(request: Request):
        return await _generate(request, False)

    @app.post(f"{API}/img2img", dependencies=[Depends(auth)])
    async def img2img(request: Request):
        return await _generate(request, True)

    @app.get(f"{API}/memory", dependencies=[Depends(auth)])
    def memory():
        """shape read at reference worker.py:327-331: response['cuda']['system']['free'|'total'] (bytes)"""
        import torch
        try:
            free = total = 0
            for w in pool.workers:
                f, t = torch.cuda.mem_get_info(w.device_index)
                free, total = free + f, total + t
            cuda = {"system": {"free": free, "used": total - free, "total": total}}
        except Exception as e:
            cuda = {"error": f"{e}"}
        try:
            import psutil
            vm = psutil.virtual_memory()
            ram = {"free": vm.available, "used": vm.used, "total": vm.total}
        except Exception as e:  # pragma: no cover
            ram = {"error": f"{e}"}
        return {"ram": ram, "cuda": cuda}

    @app.get(f"{API}/options", dependencies=[Depends(auth)])
    def get_options():
        return app.state.options

    @app.post(f"{API}/options", dependencies=[Depends(auth)])
    async def set_options(request: Request):
        """weights are resident: record what the master believes is loaded (reference worker.py:665-668)"""
        body = await request.json()
        if isinstance(body, dict):
            for k in ("sd_model_checkpoint", "sd_vae"):
                if k in body:
                    app.state.options[k] = body[k]
        return None

    @app.post(f"{API}/interrupt", dependencies=[Depends(auth)])
    def interrupt():
        pool.interrupt()
        return {}

    @app.post(f"{API}/refresh-checkpoints", dependencies=[Depends(auth)])
    def refresh_checkpoints():
        return None

    @app.post(f"{API}/refresh-loras", dependencies=[Depends(auth)])
    def refresh_loras():
        from b200sd import factory
        factory.refresh_loras()
        return None

    @app.get(f"{API}/sd-models", dependencies=[Depends(auth)])
    def sd_models():
        name = model_title.split(" [")[0]
        return [{"title": model_title, "model_name": name.rsplit(".", 1)[0], "hash": None, "sha256": None,
                 "filename": name, "config": None}]

    @app.get(f"{API}/script-info", dependencies=[Depends(auth)])
    def script_info():
        """no alwayson scripts run on this executor: the master drops all of them from the payload (worker.py:375-404)"""
        return []

    @app.post(f"{API}/server-restart", dependencies=[Depends(auth)])
    def server_restart():
        pool.restart()
        return {}

    return app


def main():  # pragma: no cover - manual entry point
    import uvicorn
    from b200sd.factory import default_engine_factory
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--host", default="0.0.0.0")
    ap.add_argument("--port", type=int, default=7860)
    ap.add_argument("--devices", default="0", help="comma-separated CUDA device indices served by this process")
    ap.add_argument("--api-auth", default=None, help="user:password (HTTP basic), like sdwui's --api-auth")
    a = ap.parse_args()
    app = create_app(default_engine_factory, [int(d) for d in a.devices.split(",")], api_auth=a.api_auth)
    uvicorn.run(app, host=a.host, port=a.port, log_level="warning")


if __name__ == "__main__":  # pragma: no cover
    main()
