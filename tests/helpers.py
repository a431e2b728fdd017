"""Shared test helpers: golden fixture loading, config parsing, per-case result logs."""
import ast
import json
import os
import tempfile

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def log_jsonl(name, payload):
    """Append one JSON row to <name> in $PB200_TEST_LOG_DIR (default: paella_b200_test_logs under the system temp directory)."""
    d = os.environ.get("PB200_TEST_LOG_DIR") or os.path.join(tempfile.gettempdir(), "paella_b200_test_logs")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, name), "a") as f:
        f.write(json.dumps(payload) + "\n")


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, name), allow_pickle=False)
    data = {k: z[k] for k in z.files}
    sd = {k[3:]: torch.from_numpy(v.copy()) for k, v in data.items() if k.startswith("sd:")}
    rest = {k: v for k, v in data.items() if not k.startswith("sd:")}
    cfg = ast.literal_eval(str(rest.pop("cfg_json"))) if "cfg_json" in rest else None
    return cfg, sd, rest


def t(a):
    return torch.from_numpy(np.asarray(a).copy())


def oracle_cfg(cfg_dict):
    from oracle.paella_oracle import PaellaConfig
    d = {k: v for k, v in cfg_dict.items() if k != "dropout"}
    return PaellaConfig(**d)
