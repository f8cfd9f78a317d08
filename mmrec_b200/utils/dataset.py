"""Interaction dataset with the reference's on-disk format and API (`src/utils/dataset.py:21-133`):
`<data_path>/<dataset>/<inter_file_name>` TSV with the user, item and `x_label` (0 train / 1 valid / 2 test) columns."""
import os

import numpy as np
import pandas as pd


class RecDataset(object):
    def __init__(self, config, df=None):
        self.config = config
        self.dataset_name = config["dataset"]
        self.dataset_path = os.path.abspath(config["data_path"] + self.dataset_name)
        self.uid_field = config["USER_ID_FIELD"]
        self.iid_field = config["ITEM_ID_FIELD"]
        self.splitting_label = config["inter_splitting_label"]
        if df is not None:
            self.df = df
            return
        path = os.path.join(self.dataset_path, config["inter_file_name"])
        if not os.path.isfile(path):
            raise ValueError("File {} not exist".format(path))
        cols = [self.uid_field, self.iid_field, self.splitting_label]
        self.df = pd.read_csv(path, usecols=cols, sep=config["field_separator"])
        self.item_num = int(self.df[self.iid_field].values.max()) + 1
        self.user_num = int(self.df[self.uid_field].values.max()) + 1

    def split(self):
        parts = []
        for label in range(3):
            part = self.df[self.df[self.splitting_label] == label].drop(columns=[self.splitting_label])
            parts.append(part)
        if self.config["filter_out_cod_start_users"]:       # users unseen in training are dropped from val/test
            train_users = np.unique(parts[0][self.uid_field].values)
            for i in (1, 2):
                parts[i] = parts[i][parts[i][self.uid_field].isin(train_users)]
        return [self.copy(p) for p in parts]

    def copy(self, new_df):
        nxt = RecDataset(self.config, new_df)
        nxt.item_num, nxt.user_num = self.item_num, self.user_num
        return nxt

    def get_user_num(self):
        return self.user_num

    def get_item_num(self):
        return self.item_num

    def shuffle(self):
        self.df = self.df.sample(frac=1, replace=False).reset_index(drop=True)

    def __len__(self):
        return len(self.df)

    def __getitem__(self, idx):
        return self.df.iloc[idx]

    def __str__(self):
        self.inter_num = len(self.df)
        nu, ni = self.df[self.uid_field].nunique(), self.df[self.iid_field].nunique()
        info = [self.dataset_name, f"The number of users: {nu}", f"Average actions of users: {self.inter_num / max(nu, 1)}",
                f"The number of items: {ni}", f"Average actions of items: {self.inter_num / max(ni, 1)}",
                f"The number of inters: {self.inter_num}",
                f"The sparsity of the dataset: {(1 - self.inter_num / max(nu, 1) / max(ni, 1)) * 100}%"]
        return "\n".join(info)

    __repr__ = __str__
