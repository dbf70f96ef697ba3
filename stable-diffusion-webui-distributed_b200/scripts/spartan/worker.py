"""Worker node model: state machine, ETA model, benchmark loop and the request boundary.

Drop-in for the reference's scripts/spartan/worker.py (`State` :36-41, `Worker` :51, `eta` :230-286,
`request` :288-504, `benchmark` :506-575, `set_state` :719-758) with the same attributes and method signatures.
`Worker` keeps the HTTP transport so an sdwui instance on another box can still be driven; the GPU-native
transport is `LocalGPUWorker` (local_worker.py), which overrides `request()` with an in-process executor.

Conscious fixes of reference quirks (SURVEY.md App. E), everything else behaves identically:
  * the scheme/trailing slash are stripped from the address that is actually stored (worker.py:107 vs :139-147)
  * the ETA-error window keeps the newest 5 samples (the reference drops new samples once it holds 5, :487-490)
"""
import base64
import copy
import io
import json
import math
import queue
import re
import time
from enum import Enum
from threading import Thread
from typing import List, Union

import requests
from modules.shared import cmd_opts
from modules.shared import state as master_state

from . import shared as sh
from .pmodels import Worker_Model
from .shared import LOG_LEVEL, logger

try:  # sdwui before / after commit 95821f0
    from webui import server_name
except ImportError:
    from modules.initialize_util import gradio_server_name

    server_name = gradio_server_name()


class InvalidWorkerResponse(Exception):
    """A worker answered with something the dispatcher cannot use."""


class State(Enum):
    IDLE = 1
    WORKING = 2
    INTERRUPTED = 3
    UNAVAILABLE = 4
    DISABLED = 5


# allowed set_state() moves: current -> targets
_TRANSITIONS = {
    State.IDLE: (State.IDLE, State.WORKING),
    State.WORKING: (State.WORKING, State.IDLE, State.INTERRUPTED),
    State.UNAVAILABLE: (State.IDLE,),
    State.INTERRUPTED: (State.WORKING,),
}


def pil_to_64(image) -> str:
    buf = io.BytesIO()
    image.save(buf, format="PNG")
    return "data:image/png;base64," + base64.b64encode(buf.getvalue()).decode("utf-8")


class Worker:
    """One node of the world (the local master, a remote sdwui, or — subclassed — a local GPU)."""

    # speed of each sampler relative to Euler a in percent (positive = faster); ETA model constants
    other_to_euler_a = {
        "DPM++ 2S a Karras": -45.87, "Euler": 4.92, "LMS": 12.66, "Heun": -40.24, "DPM2": -42.50, "DPM2 a": -46.60,
        "DPM++ 2S a": -37.10, "DPM++ 2M": 7.46, "DPM++ SDE": -39.45, "DPM fast": 15.54, "DPM adaptive": -61.40,
        "LMS Karras": 5, "DPM2 Karras": -41, "DPM2 a Karras": -38.81, "DPM++ 2M Karras": 16.20,
        "DPM++ SDE Karras": -39.71, "DDIM": 0, "PLMS": 9.31,
    }

    def __init__(self, address: Union[str, None] = None, port: int = 7860, label: Union[str, None] = None,
                 verify_remotes: bool = True, master: bool = False, tls: bool = False, state: State = State.IDLE,
                 avg_ipm: float = 0.0, eta_percent_error=None, user: str = None, password: str = None,
                 pixel_cap: int = -1):
        self.eta_percent_error = [] if eta_percent_error is None else eta_percent_error
        self.avg_ipm = avg_ipm
        self.state = state if isinstance(state, State) else State(state)
        self.address = address
        self.port = port
        self.label = label
        self.tls = tls
        self.pixel_cap = pixel_cap
        self.response = None
        self.response_time = None
        self.loaded_model = ""
        self.loaded_vae = ""
        self.supported_scripts = {}
        self.model_override: Union[str, None] = None
        self.free_vram = 0
        self.queried = False
        self.benchmarked = False
        self.jobs_requested = 0
        self.master = bool(master)
        if self.master:
            self.label = "master"
            self.address = server_name if server_name is not None else "localhost"
            self.port = 7860 if cmd_opts.port is None else cmd_opts.port
            return
        if address is None:
            raise InvalidWorkerResponse("Worker address cannot be None")
        self._normalise_address(address)
        self.user = str(user)
        self.password = str(password)
        self._open_session(verify_remotes)

    def _normalise_address(self, address: str):
        if address.startswith("http://"):
            address = address[len("http://"):]
        elif address.startswith("https://"):
            address = address[len("https://"):]
            self.tls = True
            self.port = 443
        self.address = address.rstrip("/") if address.endswith("/") else address

    def _open_session(self, verify: bool):
        self.session = requests.Session()
        self.session.auth = (self.user, self.password)
        self.session.verify = verify

    # ------------------------------------------------------------------ identity
    def __str__(self):
        return f"{self.address}:{self.port}"

    def __repr__(self):
        return f"'{self.label}'@{self.address}:{self.port}, speed: {self.avg_ipm} ipm, state: {self.state}"

    def __eq__(self, other):
        return isinstance(other, Worker) and other.label == self.label

    __hash__ = None

    @property
    def model(self) -> Worker_Model:
        return Worker_Model.from_worker(self)

    def full_url(self, route: str) -> str:
        return f"{'https' if self.tls else 'http'}://{self}/sdapi/v1/{route}"

    # ------------------------------------------------------------------ ETA model (reference worker.py:176-286)
    def eta_mpe(self):
        """mean of the stored ETA percent errors (0 when none)."""
        if not self.eta_percent_error:
            return 0
        total = 0
        for pct in self.eta_percent_error:
            total += pct
        return total / len(self.eta_percent_error)

    def eta_hr(self, payload: dict) -> float:
        """ETA of the hires-fix second pass: same model on the upscaled size and the second-pass step count."""
        second = copy.copy(payload)
        second["enable_hr"] = False
        if second["hr_second_pass_steps"] != 0:
            second["steps"] = second["hr_second_pass_steps"]
        second["width"] = math.floor(second["width"] * second["hr_scale"])
        second["height"] = math.floor(second["height"] * second["hr_scale"])
        return self.eta(payload=second, quiet=True)

    def eta(self, payload: dict, quiet: bool = False, batch_size: int = None, samples: int = None) -> float:
        """seconds this worker is predicted to need for `payload` (ipm x steps x pixels x sampler % x MPE)."""
        bench = sh.benchmark_payload
        steps = payload["steps"] if samples is None else samples
        images = payload["batch_size"] if batch_size is None else batch_size
        eta = (images / self.avg_ipm) * 60
        eta = eta * (steps / bench.steps)
        if payload.get("enable_hr", False):
            eta += self.eta_hr(payload=payload)
        eta = eta * ((payload["width"] * payload["height"]) / (bench.width * bench.height))
        sampler = payload.get("sampler_name", "Euler a")
        if sampler != "Euler a":
            pct = self.other_to_euler_a.get(sampler)
            if pct is None:
                logger.warning(f"Efficiency of sampler '{sampler}' has not been recorded.\n")
            elif pct > 0:
                eta -= eta * abs(pct / 100)
            else:
                eta += eta * abs(pct / 100)
        if len(self.eta_percent_error) > 0:
            correction = eta * (self.eta_mpe() / 100)
            if not quiet:
                logger.debug(f"correcting '{self.label}'s ETA: {eta:.2f}s -> {eta - correction:.2f}s")
            eta -= correction
        return eta

    def record_eta_error(self, predicted: float, actual: float):
        """keeps the newest 5 percent errors; |error| >= 500 % is treated as an outlier and ignored."""
        variance = ((predicted - actual) / actual) * 100
        logger.debug(f"Worker '{self.label}'s ETA was off by {variance:.2f}% (predicted {predicted:.2f}s, "
                     f"actual {actual:.2f}s)")
        if abs(variance) >= 500:
            logger.warning(f"Variance of {variance:.2f}% exceeds threshold of 500%. Ignoring...\n")
            return
        self.eta_percent_error.append(variance)
        del self.eta_percent_error[:-5]

    # ------------------------------------------------------------------ request boundary (HTTP transport)
    def _wait_for_idle(self, max_wait: int = 30):
        """a still-WORKING node may be loading weights: wait up to 30 s before a consecutive request."""
        if self.jobs_requested == 0:
            return
        waited = 0
        while self.state == State.WORKING and waited < max_wait:
            time.sleep(1)
            waited += 1
        if waited:
            logger.debug(f"waited {waited}s for worker '{self.label}' to IDLE before consecutive request")

    def _query_memory_once(self):
        if self.queried:
            return
        self.queried = True
        info = self.session.get(self.full_url("memory")).json()
        try:
            mem = info["cuda"]["system"]
            self.free_vram = mem["free"]
            logger.debug(f"Worker '{self.label}' {int(mem['free']) / 2**30:.2f}/{int(mem['total']) / 2**30:.2f} GB VRAM free\n")
        except KeyError:
            err = info.get("cuda", {}).get("error") if isinstance(info, dict) else None
            if err is not None:
                logger.warning(f"CUDA seems unavailable for worker '{self.label}'\nError: {err}")
            else:
                logger.error(f"An error occurred querying memory statistics from worker '{self.label}'\n{info}")

    def _scrub_payload(self, payload: dict) -> str:
        """make the payload JSON-serialisable in place; returns 'txt2img' or 'img2img'."""
        s_tmax = payload.get("s_tmax", 0.0)
        if s_tmax is not None and s_tmax > 1e308:
            payload["s_tmax"] = 1e308
        for cache in ("cached_uc", "cached_c", "uc", "c", "cached_hr_c", "cached_hr_uc"):
            payload.pop(cache, None)
        mode = "txt2img"
        if payload.get("init_images", None) is not None:
            mode = "img2img"
            payload["init_images"] = [pil_to_64(im) for im in payload["init_images"]]
        scripts = payload.get("alwayson_scripts", None)
        if scripts is not None:
            payload["alwayson_scripts"] = self._compatible_scripts(scripts, mode)
        mask = payload.get("image_mask", None)
        if mask is not None:
            payload["mask"] = pil_to_64(mask)
            del payload["image_mask"]
        try:
            json.dumps(payload)
        except Exception:
            logger.error(f"Failed to serialize payload: \n{payload}")
            raise
        return mode

    def _compatible_scripts(self, local_scripts: dict, mode: str) -> dict:
        if len(self.supported_scripts) <= 0:
            return {}
        remote = [s.lower() for s in self.supported_scripts[mode]]
        keep, missing = {}, []
        for name, args in local_scripts.items():
            if name.lower() in remote:
                keep[name] = args
            elif name.lower() != "distribute":
                missing.append(name)
        if missing:
            msg = "local script(s): " + ", ".join(f"[{m}]" for m in missing) + \
                  f" seem to be unsupported by worker '{self.label}'\n"
            if LOG_LEVEL == "DEBUG":
                logger.debug(msg)
            elif self.jobs_requested < 1:
                logger.warning(msg)
        return keep

    def _post_preemptible(self, route: str, payload: dict):
        """POST on an inner thread; forward a host interrupt once while waiting (0.5 s poll quantum)."""
        if payload.get("sampler_index", None) is None and payload.get("sampler_name", None) is not None:
            payload["sampler_index"] = payload["sampler_name"]
        box = queue.Queue()

        def post():
            try:
                box.put(self.session.post(self.full_url(route), json=payload))
            except Exception as e:  # forwarded to the caller's thread
                box.put(e)

        t = Thread(target=post)
        t.start()
        interrupting = False
        while t.is_alive():
            if not interrupting and master_state.interrupted is True:
                self.interrupt()
                interrupting = True
            time.sleep(0.5)
        result = box.get()
        if isinstance(result, Exception):
            raise result
        return result

    def request(self, payload: dict, option_payload: dict, sync_options: bool):
        """Run one job on this worker.  Result by side effect: self.response (dict | None), self.response_time,
        self.state, self.jobs_requested (reference worker.py:288-504)."""
        eta = None
        try:
            self._wait_for_idle()
            self.set_state(State.WORKING)
            self._query_memory_once()
            if sync_options is True:
                self.load_options(model=option_payload["sd_model_checkpoint"], vae=option_payload["sd_vae"])
            if self.benchmarked:
                eta = self.eta(payload=payload) * payload["n_iter"]
                logger.debug(f"worker '{self.label}' predicts it will take {eta:.3f}s to generate "
                             f"{payload['batch_size'] * payload['n_iter']} image(s) at {self.avg_ipm:.2f} ipm\n")
            try:
                mode = self._scrub_payload(payload)
                start = time.time()
                response = self._post_preemptible(mode, payload)
                self.response = response.json()
                if response.status_code != 200:
                    if response.status_code == 404 and self.response["detail"] == "Sampler not found":
                        logger.warning(f"falling back to Euler A sampler for worker {self.label}\n"
                                       f"this may mean you should update this worker")
                        payload["sampler_index"] = payload["sampler_name"] = "Euler a"
                        retry = Thread(target=self.request, args=(payload, option_payload, sync_options,))
                        retry.start()
                        retry.join()
                        return
                    logger.error(f"'{self.label}' response: Code <{response.status_code}> {str(response.content, 'utf-8')}")
                    self.response = None
                    raise InvalidWorkerResponse()
                if self.benchmarked and self.state != State.INTERRUPTED:
                    self.response_time = time.time() - start
                    self.record_eta_error(eta, self.response_time)
            except Exception as e:
                self.set_state(State.IDLE)
                raise InvalidWorkerResponse(e)
        except requests.RequestException:
            self.set_state(State.UNAVAILABLE)
            return
        self.set_state(State.IDLE)
        self.jobs_requested += 1

    # ------------------------------------------------------------------ benchmark (reference worker.py:506-575)
    def benchmark(self, sample_function: callable = None) -> float:
        """images per minute = mean of `samples` timed generations of sh.benchmark_payload after `warmup_samples`."""
        if self.state in (State.DISABLED, State.UNAVAILABLE):
            logger.debug(f"worker '{self.label}' is unavailable or disabled, refusing to benchmark")
            return 0
        if self.master and sample_function is None:
            logger.critical("no function provided for benchmarking master")
            return -1
        rates: List[float] = []
        for i in range(sh.samples + sh.warmup_samples):
            if self.state == State.UNAVAILABLE:
                return 0
            if callable(sample_function):
                elapsed = sample_function()
            else:
                begin = time.time()
                t = Thread(target=self.request, args=(dict(sh.benchmark_payload), None, False,),
                           name=f"{self.label}_benchmark_request")
                t.start()
                t.join()
                elapsed = time.time() - begin
            ipm = sh.benchmark_payload.batch_size / (elapsed / 60)
            if i >= sh.warmup_samples:
                logger.info(f"Sample {i - sh.warmup_samples + 1}: Worker '{self.label}'({self}) - {ipm:.2f} image(s) per minute\n")
                rates.append(ipm)
        self.avg_ipm = sum(rates) / sh.samples
        logger.debug(f"Worker '{self.label}' average ipm: {self.avg_ipm:.2f}")
        self.response = None
        self.benchmarked = True
        self.eta_percent_error = []
        self.set_state(State.IDLE)
        return self.avg_ipm

    # ------------------------------------------------------------------ misc REST utilities
    def refresh_checkpoints(self):
        try:
            for route, what in (("refresh-checkpoints", "models"), ("refresh-loras", "LORA's")):
                r = self.session.post(self.full_url(route))
                if r.status_code != 200:
                    logger.error(f"Failed to refresh {what} for worker '{self.label}'\nCode <{r.status_code}>")
        except requests.exceptions.ConnectionError:
            self.set_state(State.UNAVAILABLE)

    def interrupt(self):
        try:
            if self.session.post(self.full_url("interrupt")).status_code == 200:
                self.set_state(State.INTERRUPTED)
                logger.debug(f"successfully interrupted worker {self.label}")
        except requests.exceptions.ConnectionError:
            self.set_state(State.UNAVAILABLE)

    def reachable(self) -> bool:
        try:
            self.response = self.session.get(self.full_url("memory"), timeout=3)
            return self.response.status_code == 200
        except requests.exceptions.ConnectionError as e:
            logger.error(e)
        except requests.ReadTimeout as e:
            logger.critical(f"worker '{self.label}' is online but not responding (crashed?)")
            logger.error(e)
        return False

    def available_models(self) -> List[str]:
        if self.master or self.state in (State.UNAVAILABLE, State.DISABLED):
            return []
        url = self.full_url("sd-models")
        try:
            r = self.session.get(url=url, timeout=5)
            if r.status_code != 200:
                logger.error(f"request to {url} returned {r.status_code}")
                return []
            return [m["title"] for m in r.json()]
        except requests.RequestException:
            self.set_state(State.UNAVAILABLE)
            return []

    def load_options(self, model, vae=None):
        """POST /options with the checkpoint (hash suffix stripped) and VAE; blocks while the remote loads weights."""
        if self.master:
            return
        if self.model_override is not None:
            model = self.model_override
        name = re.sub(r"\s?\[[^]]*]$", "", model)
        body = {"sd_model_checkpoint": name}
        if vae is not None:
            body["sd_vae"] = vae
        before = self.state
        self.set_state(State.WORKING, expect_cycle=True)
        begin = time.time()
        try:
            response = self.session.post(self.full_url("options"), json=body)
        except requests.exceptions.RequestException:
            self.set_state(State.UNAVAILABLE)
            logger.error(f"failed to load options for worker '{self.label}' (connection error... OOM?)")
            return
        if before != State.WORKING:
            self.set_state(State.IDLE)
        if response.status_code == 200:
            logger.debug(f"worker '{self.label}' loaded weights in {time.time() - begin:.2f}s")
            self.loaded_model = name
            if vae is not None:
                self.loaded_vae = vae
        else:
            logger.debug(f"failed to load options for worker '{self.label}'")
        self.response = response
        return self

    def restart(self) -> bool:
        if self.master:
            return True
        try:
            r = self.session.post(self.full_url("server-restart"), timeout=3)
        except requests.ConnectionError:
            logger.info(f"worker '{self.label}' is restarting")  # sdwui drops the connection while restarting
            return True
        except requests.RequestException as e:
            logger.error(f"could not restart worker '{self.label}':\n{e}")
            return False
        if r.status_code == 200:
            logger.info(f"worker '{self.label}' is restarting")
            return True
        if r.status_code == 404:
            logger.error(f"try adding --api-server-stop to '{self.label}'s launch arguments (couldn't restart)")
        else:
            logger.error(f"could not restart worker '{self.label}': {r}")
        return False

    # ------------------------------------------------------------------ state machine (reference worker.py:719-758)
    def set_state(self, state: State, expect_cycle: bool = False):
        """Move to `state` if the FSM allows it; UNAVAILABLE is reachable from anywhere except DISABLED."""
        before = self.state

        def move(target):
            if target == self.state and not expect_cycle:
                logger.debug(f"{self.label}: potentially redundant transition {self.state.name} -> {target.name}")
                return
            logger.debug(f"{self.label}: {self.state.name} -> {target.name}")
            self.state = target

        if state in _TRANSITIONS.get(self.state, ()):
            move(state)
        if state == State.UNAVAILABLE:
            if self.state == State.DISABLED:
                logger.debug(f"worker '{self.label}' is disabled... refusing to mark as unavailable")
            else:
                logger.error(f"worker '{self.label}' at {self} was unreachable and will be avoided until reconnection")
                self.loaded_model = None  # force a model re-sync when it comes back
                self.loaded_vae = None
                move(state)
        if self.state == before and self.state != state:
            logger.debug(f"{self.label}: invalid transition {self.state.name} -> {state.name}")
