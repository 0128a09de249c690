"""utils/helpers.py surface used by the trainers: parse_arguments / get_args (Isaac-Gym flavoured
CLI: --sim_device, --pipeline, --headless, --num_envs, --use_warp) and class_to_dict."""
import argparse


def _strtobool(x):
    return str(x).lower() in ("1", "true", "t", "yes", "y", "on")


def parse_device_str(device_str):
    """isaacgym.gymutil.parse_device_str: 'cuda:1' -> ('cuda', 1); 'cpu' -> ('cpu', 0)."""
    parts = str(device_str).split(":")
    if parts[0] not in ("cpu", "cuda"):
        raise ValueError(f"Invalid device string {device_str!r}")
    return parts[0], (int(parts[1]) if len(parts) > 1 else 0)


def class_to_dict(obj) -> dict:
    if not hasattr(obj, "__dict__"):
        return obj
    out = {}
    for key in dir(obj):
        if key.startswith("_"):
            continue
        val = getattr(obj, key)
        out[key] = [class_to_dict(v) for v in val] if isinstance(val, list) else class_to_dict(val)
    return out


def parse_arguments(description="H100 aerial gym", headless=False, no_graphics=False, custom_parameters=[]):
    p = argparse.ArgumentParser(description=description)
    if headless:
        p.add_argument("--headless", action="store_true")
    if no_graphics:
        p.add_argument("--nographics", action="store_true")
    p.add_argument("--sim_device", type=str, default="cuda:0")
    p.add_argument("--pipeline", type=str, default="gpu")
    p.add_argument("--graphics_device_id", type=int, default=0)
    p.add_argument("--num_threads", type=int, default=0)
    p.add_argument("--subscenes", type=int, default=0)
    p.add_argument("--slices", type=int)
    for a in custom_parameters:
        if "name" in a and ("type" in a or "action" in a):
            kw = {"help": a.get("help", "")}
            if "type" in a:
                kw["type"] = a["type"]
                if "default" in a:
                    kw["default"] = a["default"]
            else:
                kw["action"] = a["action"]
            p.add_argument(a["name"], **kw)
    args, unknown = p.parse_known_args()
    args.sim_device_type, args.compute_device_id = parse_device_str(args.sim_device)
    if args.sim_device_type != "cuda":
        raise ValueError("sim_device=cpu: this build has no CPU pipeline (the reference's Isaac Gym CPU path is not reproduced)")
    args.use_gpu_pipeline = args.pipeline.lower() in ("gpu", "cuda")
    args.physics_engine = 1  # gymapi.SIM_PHYSX, kept as data
    args.use_gpu = True
    if no_graphics and getattr(args, "nographics", False):
        args.headless = True
    if args.slices is None:
        args.slices = args.subscenes
    return args


def get_args(additional_parameters=[]):
    custom = [
        {"name": "--headless", "type": _strtobool, "default": False, "help": "Force display off at all times"},
        {"name": "--num_envs", "type": int, "default": 64, "help": "Number of environments to create."},
        {"name": "--use_warp", "type": _strtobool, "default": True, "help": "Use ray-cast sensors"},
    ]
    args = parse_arguments(description="RL Policy", custom_parameters=custom + additional_parameters)
    args.sim_device_id = args.compute_device_id
    args.sim_device = f"{args.sim_device_type}:{args.sim_device_id}"
    return args
