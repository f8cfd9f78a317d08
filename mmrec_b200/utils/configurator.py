"""Layered YAML configuration with the reference's semantics (`src/utils/configurator.py:46-129`):
overall.yaml < dataset/<name>.yaml < model/<Name>.yaml < config_dict; `hyper_parameters` lists accumulate;
missing keys read as None.  YAML files live in `mmrec_b200/configs/` (override with `config_dir`) instead of
`./configs` relative to the CWD."""
import os
import re

import torch
import yaml

_HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_FLOAT = re.compile(r"""^(?:[-+]?(?:[0-9][0-9_]*)\.[0-9_]*(?:[eE][-+]?[0-9]+)?
    |[-+]?(?:[0-9][0-9_]*)(?:[eE][-+]?[0-9]+)|\.[0-9_]+(?:[eE][-+][0-9]+)?
    |[-+]?\.(?:inf|Inf|INF)|\.(?:nan|NaN|NAN))$""", re.X)


class _Loader(yaml.FullLoader):
    pass


# the reference widens YAML's float syntax so that `1e-05` parses as a number (configurator.py:92-104)
_Loader.add_implicit_resolver("tag:yaml.org,2002:float", _FLOAT, list("-+0123456789."))


class Config(object):
    def __init__(self, model=None, dataset=None, config_dict=None, mg=False, config_dir=None):
        config_dict = dict(config_dict or {})
        config_dict["model"], config_dict["dataset"] = model, dataset
        self.config_dir = config_dir or os.path.join(_HERE, "configs")
        merged, hyper = {}, []
        files = [os.path.join(self.config_dir, "overall.yaml"),
                 os.path.join(self.config_dir, "dataset", f"{dataset}.yaml"),
                 os.path.join(self.config_dir, "model", f"{model}.yaml")]
        if mg:
            files.append(os.path.join(self.config_dir, "mg.yaml"))
        for f in files:
            if os.path.isfile(f):
                with open(f, "r", encoding="utf-8") as fh:
                    data = yaml.load(fh.read(), Loader=_Loader) or {}
                hyper.extend(data.get("hyper_parameters") or [])
                merged.update(data)
        merged["hyper_parameters"] = hyper
        merged.update(config_dict)
        self.final_config_dict = merged
        metric = merged["valid_metric"].split("@")[0]
        merged["valid_metric_bigger"] = metric not in ("rmse", "mae", "logloss")
        if "seed" not in merged["hyper_parameters"]:
            merged["hyper_parameters"] += ["seed"]
        use_gpu = merged["use_gpu"]
        merged["device"] = torch.device("cuda" if torch.cuda.is_available() and use_gpu else "cpu")

    def __setitem__(self, key, value):
        if not isinstance(key, str):
            raise TypeError("index must be a str.")
        self.final_config_dict[key] = value

    def __getitem__(self, item):
        return self.final_config_dict.get(item)

    def __contains__(self, key):
        if not isinstance(key, str):
            raise TypeError("index must be a str.")
        return key in self.final_config_dict

    def __str__(self):
        return "\n" + "\n".join(f"{k}={v}" for k, v in self.final_config_dict.items()) + "\n\n"

    __repr__ = __str__
