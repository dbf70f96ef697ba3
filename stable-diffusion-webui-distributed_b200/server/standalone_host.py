"""Minimal stand-in for the sdwui host modules, for running the worker server OUTSIDE sdwui.

`scripts.spartan.{shared,worker,local_worker}` import `modules.shared` (cmd_opts, state) and
`modules.initialize_util` because inside sdwui they are the plugin's host.  A GPU node that only serves the REST API
has no sdwui: `install()` registers just those attributes — and nothing at all when a real `modules` package is
importable (i.e. when this code runs as an sdwui extension).
"""
import importlib.util
import os
import sys
import tempfile
import types


def install() -> bool:
    """returns True if the stand-in was installed, False if a host `modules` package already exists"""
    if "modules" in sys.modules or importlib.util.find_spec("modules") is not None:
        return False
    cfg_dir = os.environ.get("B200SD_CONFIG_DIR") or tempfile.mkdtemp(prefix="b200sd_")
    modules = types.ModuleType("modules")
    modules.__path__ = []  # a package
    shared = types.ModuleType("modules.shared")
    shared.cmd_opts = types.SimpleNamespace(
        distributed_skip_verify_remotes=True, distributed_debug=False,
        distributed_config=os.path.join(cfg_dir, "distributed-config.json"), distributed_remotes_autosave=False,
        distributed_remotes=None, port=None)
    shared.state = types.SimpleNamespace(interrupted=False, textinfo="", job_count=0, job="")
    init_util = types.ModuleType("modules.initialize_util")
    init_util.gradio_server_name = lambda: None
    modules.shared, modules.initialize_util = shared, init_util
    sys.modules.update({"modules": modules, "modules.shared": shared, "modules.initialize_util": init_util})
    return True
