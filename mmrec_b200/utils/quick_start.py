"""Run driver with the reference's flow (`src/utils/quick_start.py:19-108`): config -> dataset ->
split -> dataloaders -> hyper-parameter grid (seed reset per combination) -> model + trainer -> summary."""
import os
import platform
from itertools import product
from logging import getLogger

from ..common.trainer import Trainer
from .configurator import Config
from .dataloader import EvalDataLoader, TrainDataLoader
from .dataset import RecDataset
from .utils import dict2str, get_model, init_seed


def quick_start(model, dataset, config_dict, save_model=True, mg=False):
    config = Config(model, dataset, config_dict, mg)
    logger = getLogger()
    logger.info("██Server: \t" + platform.node())
    logger.info("██Dir: \t" + os.getcwd() + "\n")
    logger.info(config)
    data = RecDataset(config)
    logger.info(str(data))
    train_ds, valid_ds, test_ds = data.split()
    for name, ds in (("Training", train_ds), ("Validation", valid_ds), ("Testing", test_ds)):
        logger.info(f"\n===={name}====\n" + str(ds))
    train_data = TrainDataLoader(config, train_ds, batch_size=config["train_batch_size"], shuffle=True)
    valid_data = EvalDataLoader(config, valid_ds, additional_dataset=train_ds, batch_size=config["eval_batch_size"])
    test_data = EvalDataLoader(config, test_ds, additional_dataset=train_ds, batch_size=config["eval_batch_size"])

    val_metric = config["valid_metric"].lower()
    if "seed" not in config["hyper_parameters"]:
        config["hyper_parameters"] = ["seed"] + config["hyper_parameters"]
    grid = []
    for name in config["hyper_parameters"]:
        v = config[name]
        grid.append(v if isinstance(v, list) else [v])
    results, best_value, best_idx = [], 0.0, 0
    combos = list(product(*grid))
    for idx, combo in enumerate(combos):
        for name, value in zip(config["hyper_parameters"], combo):
            config[name] = value
        init_seed(config["seed"])
        logger.info("========={}/{}: Parameters:{}={}=======".format(idx + 1, len(combos), config["hyper_parameters"], combo))
        train_data.pretrain_setup()
        net = get_model(config["model"])(config, train_data).to(config["device"])
        logger.info(net)
        trainer = Trainer(config, net, mg)
        _, best_valid, best_test = trainer.fit(train_data, valid_data=valid_data, test_data=test_data, saved=save_model)
        results.append((combo, best_valid, best_test))
        if best_test[val_metric] > best_value:
            best_value, best_idx = best_test[val_metric], idx
        logger.info("best valid result: {}".format(dict2str(best_valid)))
        logger.info("test result: {}".format(dict2str(best_test)))
    logger.info("\n============All Over=====================")
    for combo, v, t in results:
        logger.info("Parameters: {}={},\n best valid: {},\n best test: {}".format(config["hyper_parameters"], combo, dict2str(v), dict2str(t)))
    logger.info("\n\n█████████████ BEST ████████████████")
    logger.info("\tParameters: {}={},\nValid: {},\nTest: {}\n\n".format(config["hyper_parameters"], results[best_idx][0],
                                                                       dict2str(results[best_idx][1]), dict2str(results[best_idx][2])))
    return results, best_idx
