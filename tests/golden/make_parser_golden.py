"""Dump the flags and defaults of the reference's command line (helper/parser.py of the PipeGCN checkout named by
PIPEGCN_REF) -> ref_parser.json."""
import importlib.util
import json
import os
import sys
from pathlib import Path

spec = importlib.util.spec_from_file_location("ref_parser", os.path.join(os.environ["PIPEGCN_REF"], "helper", "parser.py"))
mod = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mod)
sys.argv = ["main.py"]
ns = vars(mod.create_parser())
sys.argv = ["main.py", "--n_layers", "4", "--enable_pipeline", "--feat-corr", "--no-eval", "--norm", "batch"]
ns2 = vars(mod.create_parser())
out = {"defaults": ns, "parsed_example": ns2}
Path(__file__).with_name("ref_parser.json").write_text(json.dumps(out, indent=1, sort_keys=True))
print("flags:", len(ns))
