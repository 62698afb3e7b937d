"""``models.lstm`` drop-in: ``lstm`` (frame predictor) and ``gaussian_lstm`` (posterior / prior) with the
reference's constructor signatures, ``state_dict`` keys and mutable ``.hidden`` list
(reference models/lstm.py:5-44 and :46-94).  The nn layers only hold parameters; arithmetic runs in the
sm_90a kernels.  ``init_hidden`` allocates on the parameters' device instead of hard-coding ``.cuda()``."""
import torch
import torch.nn as nn


class _RecurrentBase(nn.Module):
    def __init__(self, input_size, output_size, hidden_size, n_layers, batch_size):
        super().__init__()
        self.input_size, self.output_size, self.hidden_size = input_size, output_size, hidden_size
        self.n_layers, self.batch_size = n_layers, batch_size
        self.embed = nn.Linear(input_size, hidden_size)
        self.lstm = nn.ModuleList([nn.LSTMCell(hidden_size, hidden_size) for _ in range(n_layers)])

    def init_hidden(self, batch_size=1):
        dev = self.embed.weight.device
        self.hidden = [(torch.zeros(batch_size, self.hidden_size, device=dev), torch.zeros(batch_size, self.hidden_size, device=dev))
                       for _ in range(self.n_layers)]
        return self.hidden


class lstm(_RecurrentBase):
    def __init__(self, input_size, output_size, hidden_size, n_layers, batch_size):
        super().__init__(input_size, output_size, hidden_size, n_layers, batch_size)
        self.output = nn.Sequential(nn.Linear(hidden_size, output_size), nn.Tanh())

    def forward(self, input):
        from ..infer import lstm_forward
        return lstm_forward(self, input)


class gaussian_lstm(_RecurrentBase):
    def __init__(self, input_size, output_size, hidden_size, n_layers, batch_size):
        super().__init__(input_size, output_size, hidden_size, n_layers, batch_size)
        self.mu_net = nn.Linear(hidden_size, output_size)
        self.logvar_net = nn.Linear(hidden_size, output_size)
        self.hidden = None

    def forward(self, input):
        from ..infer import gaussian_lstm_forward
        return gaussian_lstm_forward(self, input)
