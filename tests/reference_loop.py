"""A literal restatement of the reference's data pipeline and training loop, for the series-training tests and
scripts/epoch_speed.py when the reference itself is not staged: utils.py `SlidingWindowDataset` and
`create_data_loaders`, training.py `Trainer.fit` / `Trainer.evaluate` (without logging, plotting or timing)."""
import os

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset, SubsetRandomSampler


class SlidingWindowDataset(Dataset):
    """utils.py SlidingWindowDataset (horizon 1)."""

    def __init__(self, data, window, target_dim=None, horizon=1):
        self.data, self.window, self.target_dim, self.horizon = data, window, target_dim, horizon

    def __getitem__(self, index):
        x = self.data[index:index + self.window]
        y = self.data[index + self.window:index + self.window + self.horizon]
        return x, y

    def __len__(self):
        return len(self.data) - self.window


def create_data_loaders(train_dataset, batch_size, val_split=0.1, shuffle=True):
    """utils.py create_data_loaders (no test set)."""
    if val_split == 0.0:
        return DataLoader(train_dataset, batch_size=batch_size, shuffle=shuffle), None
    dataset_size = len(train_dataset)
    indices = list(range(dataset_size))
    split = int(np.floor(val_split * dataset_size))
    if shuffle:
        np.random.shuffle(indices)
    train_indices, val_indices = indices[split:], indices[:split]
    train_loader = DataLoader(train_dataset, batch_size=batch_size, sampler=SubsetRandomSampler(train_indices))
    val_loader = DataLoader(train_dataset, batch_size=batch_size, sampler=SubsetRandomSampler(val_indices))
    return train_loader, val_loader


class Trainer:
    """training.py Trainer.fit / evaluate: the per-batch host loop with sqrt(MSELoss) terms and `.item()` lists.
    `step_losses` records the per-batch (forecast, recon) values of the training batches, `epoch_times` each epoch's
    seconds (as the reference's own `epoch_times`)."""

    def __init__(self, model, optimizer, n_epochs, target_dims=None, dlpath=None, device="cuda"):
        self.model, self.optimizer, self.n_epochs = model, optimizer, n_epochs
        self.target_dims, self.dlpath, self.device = target_dims, dlpath, device
        self.forecast_criterion = torch.nn.MSELoss()
        self.recon_criterion = torch.nn.MSELoss()
        self.losses = {"train_total": [], "train_forecast": [], "train_recon": [], "val_total": [], "val_forecast": [],
                       "val_recon": []}
        self.step_losses = []
        self.epoch_times = []

    def _terms(self, x, y, preds, recons):
        if self.target_dims is not None:
            x = x[:, :, self.target_dims]
            y = y[:, :, self.target_dims].squeeze(-1)
        if preds.ndim == 3:
            preds = preds.squeeze(1)
        if y.ndim == 3:
            y = y.squeeze(1)
        return torch.sqrt(self.forecast_criterion(y, preds)), torch.sqrt(self.recon_criterion(x, recons))

    def fit(self, train_loader, val_loader=None):
        import time
        self.init_train_loss = self.evaluate(train_loader)
        if val_loader is not None:
            self.init_val_loss = self.evaluate(val_loader)
        for epoch in range(self.n_epochs):
            epoch_start = time.time()
            self.model.train()
            forecast_b_losses, recon_b_losses = [], []
            for x, y in train_loader:
                x = x.to(self.device)
                y = y.to(self.device)
                self.optimizer.zero_grad()
                preds, recons = self.model(x)
                forecast_loss, recon_loss = self._terms(x, y, preds, recons)
                loss = forecast_loss + recon_loss
                loss.backward()
                self.optimizer.step()
                forecast_b_losses.append(forecast_loss.item())
                recon_b_losses.append(recon_loss.item())
            self.step_losses += list(zip(forecast_b_losses, recon_b_losses))
            forecast_b_losses = np.array(forecast_b_losses)
            recon_b_losses = np.array(recon_b_losses)
            forecast_epoch_loss = np.sqrt((forecast_b_losses ** 2).mean())
            recon_epoch_loss = np.sqrt((recon_b_losses ** 2).mean())
            self.losses["train_forecast"].append(forecast_epoch_loss)
            self.losses["train_recon"].append(recon_epoch_loss)
            self.losses["train_total"].append(forecast_epoch_loss + recon_epoch_loss)
            if val_loader is not None:
                forecast_val_loss, recon_val_loss, total_val_loss = self.evaluate(val_loader)
                self.losses["val_forecast"].append(forecast_val_loss)
                self.losses["val_recon"].append(recon_val_loss)
                self.losses["val_total"].append(total_val_loss)
                if total_val_loss <= self.losses["val_total"][-1]:
                    self.save("model.pt")
            self.epoch_times.append(time.time() - epoch_start)
        if val_loader is None:
            self.save("model.pt")

    def evaluate(self, data_loader):
        self.model.eval()
        forecast_losses, recon_losses = [], []
        with torch.no_grad():
            for x, y in data_loader:
                x = x.to(self.device)
                y = y.to(self.device)
                preds, recons = self.model(x)
                forecast_loss, recon_loss = self._terms(x, y, preds, recons)
                forecast_losses.append(forecast_loss.item())
                recon_losses.append(recon_loss.item())
        forecast_loss = np.sqrt((np.array(forecast_losses) ** 2).mean())
        recon_loss = np.sqrt((np.array(recon_losses) ** 2).mean())
        return forecast_loss, recon_loss, forecast_loss + recon_loss

    def save(self, file_name):
        if self.dlpath is not None:
            os.makedirs(self.dlpath, exist_ok=True)
            torch.save(self.model.state_dict(), os.path.join(self.dlpath, file_name))
