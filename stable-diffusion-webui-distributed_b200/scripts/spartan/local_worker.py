"""LocalGPUWorker — a Worker whose request() runs on a GPU of this box instead of POSTing to a remote sdwui.

This is THE boundary of the build (SURVEY.md §8b): the reference's `Worker.request(payload, option_payload,
sync_options)` (scripts/spartan/worker.py:288-504) does `session.post(full_url("txt2img"|"img2img"))` (:432-435) and
stores the JSON reply in `self.response`; here the same call, with the same payload dict and the same side effects
(`self.response`, `self.response_time`, `self.state`, `self.jobs_requested`), drives a b200sd.SDEngine on
`cuda:<device_index>`.  The reply keeps the API schema read by scripts/distributed.py:78-93,:152,:347
(`images`, `parameters`, `info` JSON string) and adds `tensors` — the decoded uint8 images on the host — so the
collector can skip PNG + base64 (the reference's per-image wire format) when both sides are local.

Error mapping (reference worker.py:494-500): a CUDA / kernel-library failure marks the device UNAVAILABLE and leaves
`response = None` (the collector skips the job, distributed.py:148); anything else re-raises InvalidWorkerResponse.
"""
import base64
import io
import json
import time
from threading import Thread

import numpy as np
import torch
from modules.shared import state as master_state

from .shared import logger
from .worker import InvalidWorkerResponse, State, Worker

def supported_samplers():
    """every sampler name of the reference's ETA table (worker.py:75-94) plus Euler a — b200sd.engine.SAMPLERS"""
    from b200sd.engine import SAMPLERS
    return tuple(SAMPLERS)


class LocalGPUWorker(Worker):
    is_local_gpu = True

    def __init__(self, device_index: int, engine_factory, label: str = None, avg_ipm: float = 0.0, png_images=False,
                 **kw):
        kw.pop("address", None)
        kw.pop("port", None)
        kw.pop("verify_remotes", None)
        kw.pop("master", None)
        super().__init__(address=f"cuda:{device_index}", port=device_index, label=label or f"gpu{device_index}",
                         verify_remotes=False, avg_ipm=avg_ipm, **kw)
        self.device_index = device_index
        self.device = f"cuda:{device_index}"
        self._factory = engine_factory
        self._engine = None
        self.png_images = png_images  # also fill response["images"] with base64 PNGs (API-exact, slower)
        self.make_pil = False         # set by World when the thin-client collector will want PIL images
        self.queried = True

    # ------------------------------------------------------------------ engine access
    @property
    def engine(self):
        if self._engine is None:
            self._engine = self._factory(self.device)
        return self._engine

    # ------------------------------------------------------------------ transport overrides (no HTTP)
    def reachable(self) -> bool:
        try:
            ok = torch.cuda.is_available() and self.device_index < torch.cuda.device_count()
        except Exception:  # pragma: no cover
            ok = False
        self.response = None
        return ok

    def query_scripts(self) -> dict:
        return {"txt2img": ["controlnet"], "img2img": ["controlnet"]}

    def load_options(self, model, vae=None):
        """weights are replicated on every device at engine construction; just record what is loaded"""
        self.loaded_model, self.loaded_vae = model, vae
        return self

    def interrupt(self):
        if self._engine is not None:
            self._engine.interrupted = True
        self.set_state(State.INTERRUPTED)

    def refresh_checkpoints(self):
        """the reference posts refresh-checkpoints and refresh-loras: LoRA files are read again on their next use"""
        from b200sd import factory
        factory.refresh_loras()

    def available_models(self):
        return []

    def restart(self) -> bool:
        """reference Worker.restart posts /server-restart; here: drop the engine (weights, plans, graphs) — the next
        request rebuilds it"""
        from b200sd import factory, upscale
        factory.evict(self.device)
        upscale.evict(self.device)
        self._engine = None
        return True

    # ------------------------------------------------------------------ the request boundary
    def request(self, payload: dict, option_payload: dict, sync_options: bool):
        eta = None
        try:
            self._wait_for_idle()
            self.set_state(State.WORKING)
            if sync_options is True and option_payload is not None:
                self.load_options(model=option_payload["sd_model_checkpoint"], vae=option_payload["sd_vae"])
            if self.benchmarked:
                eta = self.eta(payload=payload) * payload.get("n_iter", 1)
            begin = time.time()
            result = {}

            def work():
                try:
                    result["response"] = self._generate(payload)
                except Exception as e:  # forwarded to the request thread
                    result["error"] = e

            t = Thread(target=work, name=f"{self.label}_generate")
            t.start()
            interrupting = False
            while t.is_alive():  # same shape as the reference's poll loop, 20 ms instead of 0.5 s
                if not interrupting and master_state.interrupted is True:
                    self.interrupt()
                    interrupting = True
                t.join(0.02)
            if "error" in result:
                raise result["error"]
            self.response = result["response"]
            if self.benchmarked and self.state != State.INTERRUPTED:
                self.response_time = time.time() - begin
                self.record_eta_error(eta, self.response_time)
        except Exception as e:
            self.response = None
            if self._is_device_failure(e):
                logger.error(f"'{self.label}' ({self.device}) failed: {e}", exc_info=logger.isEnabledFor(10))
                self.set_state(State.UNAVAILABLE)
                return
            self.set_state(State.IDLE)
            raise InvalidWorkerResponse(e)
        self.set_state(State.IDLE)
        self.jobs_requested += 1

    @staticmethod
    def _is_device_failure(e: Exception) -> bool:
        name = type(e).__name__
        return name in ("B200SDError", "OutOfMemoryError", "AcceleratorError") or \
            (isinstance(e, RuntimeError) and "CUDA" in str(e))

    def _generate(self, payload: dict) -> dict:
        from b200sd.factory import tokenize_prompts
        eng = self.engine
        eng.interrupted = False
        batch = int(payload["batch_size"])
        n_iter = int(payload.get("n_iter", 1))
        steps = int(payload["steps"])
        width, height = int(payload["width"]), int(payload["height"])
        if batch < 1 or n_iter < 1 or steps < 1:
            raise ValueError(f"batch_size {batch}, n_iter {n_iter}, steps {steps}: all must be at least 1")
        sampler = payload.get("sampler_name") or payload.get("sampler_index") or "Euler a"
        if sampler not in supported_samplers():
            logger.warning(f"falling back to Euler a sampler for worker {self.label} ('{sampler}' is not implemented)")
            sampler = "Euler a"
        scheduler = payload.get("scheduler")  # sdwui >= 1.9 sends the noise schedule separately from the sampler
        if scheduler not in (None, "", "Automatic"):
            from b200sd.engine import SCHEDULERS
            if sampler == "DDIM" or (scheduler not in SCHEDULERS and str(scheduler).lower() not in SCHEDULERS):
                if sampler != "DDIM":
                    logger.warning(f"scheduler '{scheduler}' is not implemented on worker {self.label}: using the sampler's default")
                scheduler = None
        controls = self._controls(eng, payload, width, height)
        # an inpainting checkpoint (9-channel UNet) is conditioned on the mask and the masked init image, with sdwui's
        # inpainting_mask_weight; other engines never see the setting
        mask_weight = self._inpainting_mask_weight(payload) if getattr(eng, "inpainting", False) else None
        init_u8 = None
        inpaint = None
        if payload.get("init_images"):
            init_pil = self._init_images_pil(payload["init_images"])
            mask_img = payload.get("image_mask") if payload.get("image_mask") is not None else payload.get("mask")
            if mask_img is not None:
                # inpainting (reference worker.py:365-373 sends `image_mask` as the API's `mask`, :406-410 the other fields)
                from b200sd import inpaint as inp
                from PIL import Image
                if isinstance(mask_img, str):
                    data = mask_img.split(",", 1)[1] if mask_img.startswith("data:") else mask_img
                    mask_img = Image.open(io.BytesIO(base64.b64decode(data)))
                down = 2 ** (len(eng.vae_cfg.ch_mult) - 1)   # 8 for the kl-f8 autoencoder
                blur = payload.get("mask_blur")
                kw = dict(mask_blur=4 if blur is None else int(blur), invert=bool(payload.get("inpainting_mask_invert") or 0))
                if payload.get("inpaint_full_res") not in (None, False, 0):   # "Only masked"
                    pad = payload.get("inpaint_full_res_padding")
                    inpaint = inp.prepare_mask_only_masked(mask_img, width, height, height // down, width // down,
                                                           padding=32 if pad is None else int(pad), **kw)
                    if inpaint is not None:
                        full = torch.stack([torch.from_numpy(np.array(im.convert("RGB"))) for im in
                                            (init_pil[i % len(init_pil)] for i in range(batch))])
                        inpaint_overlays = inp.overlays_for(full, inpaint)
                        init_u8 = inp.crop_init_images([init_pil[i % len(init_pil)] for i in range(batch)], inpaint)
                if inpaint is None and init_u8 is None:
                    init_u8 = self._init_images_u8(init_pil, batch, width, height)
                    if payload.get("inpaint_full_res") in (None, False, 0):
                        inpaint = inp.prepare_mask(mask_img, width, height, height // down, width // down, **kw)
                        inpaint_overlays = inp.overlays_for(init_u8, inpaint)
                if inpaint is not None:
                    fill = payload.get("inpainting_fill")
                    inpaint_fill = 1 if fill is None else int(fill)
                    if inpaint_fill == 0:   # "fill": blur the surroundings into the masked region before encoding
                        init_u8 = inp.fill_masked(init_u8, inpaint)
            else:
                init_u8 = self._init_images_u8(init_pil, batch, width, height)
        ds = payload.get("denoising_strength")
        denoise = 0.75 if ds is None else float(ds)   # an explicit 0 stays 0 (the noised init comes back untouched)
        prompt = payload.get("prompt", "") or ""
        negative = payload.get("negative_prompt", "") or ""
        seed = int(payload.get("seed", -1))
        subseed = int(payload.get("subseed", -1))
        if seed == -1:   # API default (the benchmark payload carries no seed): draw one like sdwui's fix_seed
            import random
            seed = random.randrange(4294967294)
        if subseed == -1:
            import random
            subseed = random.randrange(4294967294)
        cfg_scale = float(payload.get("cfg_scale", 7.0))
        strength = float(payload.get("subseed_strength") or 0.0)
        # sdwui extra networks: the tags leave the positive prompts before scheduling and tokenization (the infotext keeps
        # them); every named LoRA file is read, and refused if need be, before the engine changes a weight
        from b200sd import factory, lora
        body, refs = lora.parse_prompt(prompt)
        nets = factory.loras(refs, eng) if refs else []
        hires_fix = bool(payload.get("enable_hr")) and not payload.get("init_images")
        hr_body, hr_nets = body, nets
        if hires_fix and payload.get("hr_prompt"):   # sdwui hr_extra_network_data: hr_prompt's own tags
            hr_body, hr_refs = lora.parse_prompt(payload["hr_prompt"])
            hr_nets = factory.loras(hr_refs, eng) if hr_refs else []
        vocab = eng.clip_cfg.vocab
        pad = getattr(eng.clip_cfg, "pad_id", None)   # the token after each chunk's first EOS (SD 2.x: 0)
        mult_all = None
        # prompt editing / alternation: sdwui's schedules over the sampler's total steps.  A prompt whose schedule has
        # one entry is that entry's text (the prompt itself without schedule syntax) for every step.
        sched_kw, hr_kw = {}, {}
        cond_text, neg_text = body, negative
        if "prompt_tokens" not in payload:
            from b200sd.engine import total_steps
            old = self._use_old_scheduling(payload)
            base = total_steps(sampler, steps)
            cs = self._schedule(body, base, None, old, vocab, pad)
            us = self._schedule(negative, base, None, old, vocab, pad)
            if len(cs[0].ends) > 1 or len(us[0].ends) > 1:
                sched_kw["schedule"] = (cs[0], us[0])
            cond_text, neg_text = cs[1][0], us[1][0]
            if hires_fix:
                # sdwui calculate_hr_conds: hr_prompt / hr_negative_prompt (empty: the first pass's), over the hires
                # steps with the first pass's as the base of the offsets
                hires = total_steps(sampler, int(payload.get("hr_second_pass_steps") or 0) or steps)
                hc = self._schedule(hr_body, base, hires, old, vocab, pad)
                hu = self._schedule(payload.get("hr_negative_prompt") or negative, base, hires, old, vocab, pad)
                if sched_kw or len(hc[1]) > 1 or len(hu[1]) > 1 or (hc[1][0], hu[1][0]) != (cond_text, neg_text):
                    hr_kw["hr_schedule"] = (hc[0], hu[0])
        if "prompt_tokens" in payload:  # benchmark / tests hand pre-tokenised prompts through
            tok_all = torch.as_tensor(payload["prompt_tokens"]).long().reshape(-1, 77)
        else:   # sdwui prompt syntax: emphasis weights, BREAK, 77-token chunks
            tok_all, mult_all = tokenize_prompts([cond_text] * batch, vocab, pad)
        neg_all, neg_mult = tokenize_prompts([neg_text] * batch, vocab, pad)
        # emphasis multipliers reach the engine only when some weight differs from 1 (all 1 is the unweighted path)
        weighted = lambda m: m is not None and bool((m != 1.0).any())  # noqa: E731
        weights = {"neg_multipliers": neg_mult} if weighted(neg_mult) else {}
        weights.update(sched_kw)
        if controls:   # a payload without ControlNet units reaches the engine with exactly the arguments it always had
            weights["controls"] = controls
        tiling = self._tiling(payload)
        if tiling:     # likewise an untiled payload
            weights["tiling"] = True
        if mask_weight is not None:
            weights["inpainting_mask_weight"] = mask_weight
        if nets:       # likewise a payload without LoRA tags
            weights["loras"] = nets
        tome, tome_hr = self._token_merging(payload, img2img=init_u8 is not None)
        # a payload whose ratio resolves to 0 (or below: nothing is merged) reaches the engine with exactly the
        # arguments it always had
        tome_kw = {"token_merging_ratio": float(tome)} if tome > 0 else {}
        chunks = []
        for it in range(n_iter):
            # variation seeds: image k of iteration `it` blends noise(seed + k) with noise(subseed + k)
            # sdwui processing.py: all_seeds[k] = seed + (k if subseed_strength == 0 else 0), all_subseeds[k] = subseed + k
            eng.variation = (subseed + it * batch, strength) if strength != 0 else (None, 0.0)
            seed_it = seed if strength != 0 else seed + it * batch
            tok = tok_all[:batch] if tok_all.shape[0] >= batch else tok_all[:1].expand(batch, -1)
            if weighted(mult_all):
                weights["multipliers"] = mult_all[:batch]
            if init_u8 is not None:
                kw = {} if inpaint is None else {"latmask": inpaint.latmask, "inpainting_fill": inpaint_fill}
                if inpaint is not None and mask_weight is not None:   # the conditioning mask: sdwui's image_mask
                    kw["image_mask"] = torch.from_numpy(np.array(inpaint.fill_mask.convert("L")))
                u8 = eng.img2img(tok, neg_all, seed_it, init_u8, denoising_strength=denoise, steps=steps,
                                 cfg_scale=cfg_scale, sampler=sampler, scheduler=scheduler, **kw, **weights, **tome_kw)
            elif payload.get("enable_hr"):
                # hires fix (reference eta_hr, worker.py:205): second pass at hr_scale x after the hr_upscaler
                hr_scale = float(payload.get("hr_scale") or 2.0)
                if payload.get("hr_resize_x") and payload.get("hr_resize_y"):
                    hr_scale = float(payload["hr_resize_x"]) / width
                hires = dict(weights, **tome_kw, **hr_kw)
                same = lambda a, b: [(f.key, r) for f, r in a] == [(f.key, r) for f, r in b]  # noqa: E731
                if not same(hr_nets, nets):   # the second pass's own networks (none: pristine weights)
                    hires["hr_loras"] = hr_nets
                if tome_hr > 0:
                    hires["token_merging_ratio_hr"] = float(tome_hr)
                hires.update(self._hires_upscaler(payload, width, height, hr_scale))
                u8 = eng.txt2img_hires(tok, neg_all, seed_it, steps=steps, cfg_scale=cfg_scale, height=height,
                                       width=width, hr_scale=hr_scale,
                                       hr_steps=int(payload.get("hr_second_pass_steps") or 0),
                                       denoising_strength=0.7 if ds is None else float(ds), sampler=sampler,
                                       scheduler=scheduler, **hires)
            else:
                u8 = eng.txt2img(tok, neg_all, seed_it, steps=steps, cfg_scale=cfg_scale, height=height,
                                 width=width, sampler=sampler, scheduler=scheduler, **weights, **tome_kw)
            chunks.append(u8)
            if eng.interrupted:
                break
        images = torch.cat(chunks) if len(chunks) > 1 else chunks[0]
        host_chw = None
        if images.device.type == "cuda":
            with torch.cuda.device(images.device):  # this thread's current device is cuda:0 whatever the worker drives
                host = torch.empty(images.shape, dtype=torch.uint8, pin_memory=True)
                host.copy_(images, non_blocking=True)
                if inpaint is None:
                    # what the collector needs per image — CHW float in [0, 1] for `pp.images` (reference
                    # distributed.py:102-106) — is made on the device and copied out next to the bytes: the conversion
                    # of a 32-image job cost the ONE collector thread 60 ms, times the number of jobs.  +0.5: sdwui's
                    # later `(255 * x).astype(uint8)` then returns exactly these bytes.
                    chw = images.permute(0, 3, 1, 2).float().add_(0.5).div_(255.0)
                    host_chw = torch.empty(chw.shape, dtype=torch.float32, pin_memory=True)
                    host_chw.copy_(chw, non_blocking=True)
                torch.cuda.current_stream().synchronize()
        else:  # an engine double in the host-logic tests; the real engine refuses non-CUDA devices
            host = images.to(torch.uint8).contiguous()
        if inpaint is not None:   # sdwui apply_overlay: the original pixels come back through the blurred mask
            from b200sd import inpaint as inp
            host = inp.apply_overlays(host, inpaint_overlays, inpaint.paste_to)
        pil = None
        if self.make_pil:   # thin-client collector (World._bypass_local_generation): PIL objects built here, per job thread
            from PIL import Image
            pil = [Image.fromarray(host[i].numpy()) for i in range(host.shape[0])]
        n = host.shape[0]
        seeds = [seed + (i if strength == 0 else 0) for i in range(n)]
        subseeds = [subseed + i for i in range(n)]
        # sdwui create_infotext: "Conditional mask weight" when img2img runs with inpainting conditioning
        cond_weight = f", Conditional mask weight: {mask_weight}" if mask_weight is not None and init_u8 is not None else ""
        # ... then the token merging ratios (the hires one with the hires fix only), then Tiling
        if tome != 0:
            cond_weight += f", Token merging ratio: {tome}"
        if tome_hr != 0 and init_u8 is None and payload.get("enable_hr"):
            cond_weight += f", Token merging ratio hr: {tome_hr}"
        infotexts = [f"{prompt}\nNegative prompt: {negative}\nSteps: {steps}, Sampler: {sampler}, CFG scale: {cfg_scale}, "
                     f"Seed: {s}, Size: {width}x{height}" + cond_weight + (", Tiling: True" if tiling else "") for s in seeds]
        info = {"all_seeds": seeds, "all_subseeds": subseeds, "all_prompts": [prompt] * n,
                "all_negative_prompts": [negative] * n, "infotexts": infotexts, "seed": seeds[0], "subseed": subseeds[0],
                "prompt": prompt, "negative_prompt": negative}
        return {"images": [self._png_b64(host[i]) for i in range(n)] if self.png_images else [None] * n,
                "tensors": host, "tensors_chw": host_chw, "pil": pil,
                "parameters": {"batch_size": batch, "n_iter": n_iter, "steps": steps, "width": width, "height": height,
                               "sampler_name": sampler, "cfg_scale": cfg_scale, "seed": seed},
                "info": json.dumps(info)}

    def _hires_upscaler(self, payload: dict, width: int, height: int, hr_scale: float) -> dict:
        """txt2img_hires keyword arguments for the payload's hr_upscaler: none for "Latent" (the call keeps exactly its
        arguments), else the upscaler and, for ESRGAN models, sdwui's ESRGAN_tile / ESRGAN_tile_overlap settings.
        An upscaler that is not served falls back to "Latent" with a warning."""
        from b200sd import upscale
        name = payload.get("hr_upscaler") or "Latent"
        if name == "Latent":
            return {}
        try:
            kind, stem = upscale.kind(name)
            if kind != "latent" and (int(width * hr_scale) % 8 or int(height * hr_scale) % 8):
                raise upscale.UnsupportedUpscaler("the hires size is not a multiple of 8")
            if kind == "esrgan":   # load (and cache) the model now: a file that is not a 4x RRDBNet falls back
                upscale.model(stem, self.engine.device)
        except upscale.UnsupportedUpscaler as e:
            logger.warning(f"hires upscaler '{name}' is not implemented on worker {self.label} ({e}): using 'Latent'")
            return {}
        out = {"upscaler": name}
        if kind == "esrgan":
            opts = payload.get("override_settings") or {}
            if opts.get("ESRGAN_tile") is not None:
                out["upscaler_tile"] = int(opts["ESRGAN_tile"])
            if opts.get("ESRGAN_tile_overlap") is not None:
                out["upscaler_overlap"] = int(opts["ESRGAN_tile_overlap"])
        return out

    @staticmethod
    def _token_merging(payload: dict, img2img: bool):
        """(first-pass ratio, hires ratio) of sdwui's token merging for the request, as processing.get_token_merging_ratio
        resolves them; `opts.X` is override_settings["X"] if present, else the options of the sdwui this runs in, else 0.
        A non-numeric value raises ValueError."""
        overrides = payload.get("override_settings") or {}

        def num(v):
            if v is None:
                return 0
            if isinstance(v, bool) or not isinstance(v, (int, float, str)):
                raise ValueError(f"token merging ratio {v!r} is not a number")
            return float(v) if isinstance(v, str) else v   # float() raises ValueError for a non-numeric string

        def opt(name):
            if name in overrides:
                return num(overrides[name])
            import modules.shared
            return num(getattr(getattr(modules.shared, "opts", None), name, None))

        p_ratio, p_hr = num(payload.get("token_merging_ratio")), num(payload.get("token_merging_ratio_hr"))
        o_ratio, o_hr, o_img = opt("token_merging_ratio"), opt("token_merging_ratio_hr"), opt("token_merging_ratio_img2img")
        if img2img:
            return p_ratio or ("token_merging_ratio" in overrides and o_ratio) or o_img or o_ratio, 0
        return p_ratio or o_ratio, p_hr or o_hr or p_ratio or o_ratio

    @staticmethod
    def _schedule(text: str, steps: int, hires_steps, old: bool, vocab: int, pad):
        """(PromptSchedule of a prompt, its entries' texts): sdwui's schedule, every entry tokenized in one call so
        that all have the chunk count of the longest"""
        from b200sd.engine import PromptSchedule
        from b200sd.factory import tokenize_prompts
        from b200sd.prompts import prompt_schedule
        sch = prompt_schedule(text, steps, hires_steps, old)
        ids, mult = tokenize_prompts([t for _, t in sch], vocab, pad)
        return PromptSchedule([e for e, _ in sch], ids, mult if bool((mult != 1.0).any()) else None), [t for _, t in sch]

    @staticmethod
    def _use_old_scheduling(payload: dict) -> bool:
        """sdwui's use_old_scheduling option: the request's override_settings, then the options of the sdwui this runs
        in, then False"""
        value = (payload.get("override_settings") or {}).get("use_old_scheduling")
        if value is None:
            import modules.shared
            value = getattr(getattr(modules.shared, "opts", None), "use_old_scheduling", False)
        return bool(value)

    @staticmethod
    def _tiling(payload: dict) -> bool:
        """sdwui's tiling setting of the request: the payload's `tiling` unless it is None, then the request's
        override_settings, then the options of the sdwui this runs in (sdwui >= 1.6 leaves p.tiling None until
        process_images_inner reads opts.tiling; a host without that option gives False)"""
        value = payload.get("tiling")
        if value is None:
            value = (payload.get("override_settings") or {}).get("tiling")
        if value is None:
            import modules.shared
            value = getattr(getattr(modules.shared, "opts", None), "tiling", False)
        return bool(value)

    @staticmethod
    def _inpainting_mask_weight(payload: dict) -> float:
        """sdwui's inpainting_mask_weight of the request: override_settings, then the options of the sdwui this runs in,
        then 1.0; outside [0, 1] it is refused"""
        value = (payload.get("override_settings") or {}).get("inpainting_mask_weight")
        if value is None:
            import modules.shared
            value = getattr(getattr(modules.shared, "opts", None), "inpainting_mask_weight", None)
        w = 1.0 if value is None else float(value)
        if not 0.0 <= w <= 1.0:
            raise ValueError(f"inpainting_mask_weight {w} is outside [0, 1]")
        return w

    def _controls(self, eng, payload: dict, width: int, height: int):
        """the payload's enabled ControlNet units as SDEngine `controls` (None: no unit); refusals raise ValueError"""
        from b200sd import controlnet as ctl, factory
        units = ctl.parse_units(payload.get("alwayson_scripts"), width, height)
        if not units:
            return None
        if eng.unet_cfg.adm_in_channels:
            raise ValueError("ControlNet is not served for SDXL")
        if getattr(eng, "inpainting", False):
            raise ValueError("ControlNet is not served with an inpainting checkpoint")
        if payload.get("enable_hr") and not payload.get("init_images"):
            raise ValueError("ControlNet together with the hires fix is not served")
        return [(factory.controlnet(u.model, device=str(eng.device), dtype=eng.dtype), u.image, u.weight, u.start, u.end)
                for u in units]

    @staticmethod
    def _init_images_pil(init_images):
        """payload['init_images'] (PIL images, as sdwui holds them, the API's base64 PNG strings, or uint8 HWC tensors)
        -> RGB PIL images at their own size"""
        from PIL import Image
        out = []
        for item in init_images:
            if isinstance(item, str):
                data = item.split(",", 1)[1] if item.startswith("data:") else item
                item = Image.open(io.BytesIO(base64.b64decode(data)))
            if isinstance(item, torch.Tensor):
                item = Image.fromarray(item.to(torch.uint8).cpu().numpy())
            out.append(item.convert("RGB"))
        return out

    @staticmethod
    def _init_images_u8(init_images, batch: int, width: int, height: int) -> torch.Tensor:
        """RGB PIL images -> uint8 [batch, H, W, 3] at the processing size (resize_mode 0, LANCZOS); image i of the job uses
        init_images[i % len] (sdwui repeats a single init image per batch)."""
        from PIL import Image
        out = []
        for img in init_images:
            if img.size != (width, height):
                img = img.resize((width, height), Image.LANCZOS)
            out.append(torch.from_numpy(np.ascontiguousarray(np.asarray(img))))
        return torch.stack([out[i % len(out)] for i in range(batch)])

    @staticmethod
    def _png_b64(hwc_u8: torch.Tensor) -> str:
        from PIL import Image
        buf = io.BytesIO()
        Image.fromarray(hwc_u8.numpy()).save(buf, format="PNG")
        return base64.b64encode(buf.getvalue()).decode("utf-8")

    # ------------------------------------------------------------------ benchmark: measured it/s of the executor
    def benchmark(self, sample_function: callable = None) -> float:
        """Same protocol as the reference (2 warm-up + 3 timed generations of the benchmark payload, mean ipm,
        worker.py:506-575) but timed around the local executor; the first warm-up also builds plans and graphs."""
        return super().benchmark(sample_function=sample_function)
