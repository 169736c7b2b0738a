"""``mlp_field_of``: which user modules are recognised as the examples' MLP field (CPU only: the probe is host logic)."""
import torch

from torchcde_b200 import linear_field, mlp_field
from torchcde_b200.mlp_field import mlp_field_of

H, C, W = 8, 3, 16
T0 = [0.0, 1.0, 5.0]


class CDEFunc(torch.nn.Module):
    """example/time_series_classification.py:20-51."""

    def __init__(self, input_channels=C, hidden_channels=H, width=W, bias=True):
        super().__init__()
        self.input_channels, self.hidden_channels = input_channels, hidden_channels
        self.linear1 = torch.nn.Linear(hidden_channels, width, bias=bias)
        self.linear2 = torch.nn.Linear(width, input_channels * hidden_channels, bias=bias)

    def forward(self, t, z):
        z = self.linear1(z)
        z = z.relu()
        z = self.linear2(z)
        z = z.tanh()
        return z.view(z.size(0), self.hidden_channels, self.input_channels)


class MlpField(torch.nn.Module):
    """bench.py's generic-field workload."""

    def __init__(self):
        super().__init__()
        self.linear1 = torch.nn.Linear(H, W)
        self.linear2 = torch.nn.Linear(W, H * C)

    def forward(self, tt, z):
        z = self.linear2(self.linear1(z).relu()).tanh()
        return z.view(*z.shape[:-1], H, C)


class Sequential(torch.nn.Module):
    """The same field through nn.Sequential and activation modules, with the output layer declared first."""

    def __init__(self):
        super().__init__()
        self.out = torch.nn.Linear(W, H * C)
        self.inp = torch.nn.Sequential(torch.nn.Linear(H, W), torch.nn.ReLU())
        self.act = torch.nn.Tanh()

    def forward(self, t, z):
        return self.act(self.out(self.inp(z))).view(*z.shape[:-1], H, C)


class Square(torch.nn.Module):
    """C = 1 and W = H: both orderings of the two layers fit the shapes; the module applies the second one first."""

    def __init__(self):
        super().__init__()
        self.first = torch.nn.Linear(H, H)
        self.second = torch.nn.Linear(H, H)

    def forward(self, t, z):
        return torch.tanh(self.first(torch.relu(self.second(z)))).view(*z.shape[:-1], H, 1)


class WithDropout(MlpField):
    def __init__(self):
        super().__init__()
        self.drop = torch.nn.Dropout(0.5)

    def forward(self, tt, z):
        z = self.linear2(self.drop(self.linear1(z).relu())).tanh()
        return z.view(*z.shape[:-1], H, C)


class ModeDependent(MlpField):
    """No extra submodule, but the forward itself branches on the training flag."""

    def forward(self, tt, z):
        out = super().forward(tt, z)
        return out * 0.5 if self.training else out


def _variant(body):
    class Variant(MlpField):
        def forward(self, tt, z):
            return body(self, tt, z).view(*z.shape[:-1], H, C)
    return Variant()


REJECTED = {
    "softplus": lambda m, t, z: m.linear2(torch.nn.functional.softplus(m.linear1(z))).tanh(),
    "sigmoid": lambda m, t, z: m.linear2(torch.sigmoid(m.linear1(z))).tanh(),
    "no_tanh": lambda m, t, z: m.linear2(m.linear1(z).relu()),
    "depends_on_t": lambda m, t, z: m.linear2(m.linear1(z).relu()).tanh() * (1 + 0.1 * t),
    "scaled_output": lambda m, t, z: 2 * m.linear2(m.linear1(z).relu()).tanh(),
}


def _z0(batch=5):
    return torch.randn(batch, H, generator=torch.Generator().manual_seed(1))


def test_the_examples_field_is_recognised():
    torch.manual_seed(0)
    func = CDEFunc()
    got = mlp_field_of(func, _z0(), C, T0)
    assert got is not None
    assert got[0] is func.linear1.weight and got[1] is func.linear1.bias
    assert got[2] is func.linear2.weight and got[3] is func.linear2.bias
    assert mlp_field_of(MlpField(), _z0(), C, T0) is not None


def test_layers_without_bias_are_recognised():
    torch.manual_seed(0)
    func = CDEFunc(bias=False)
    got = mlp_field_of(func, _z0(), C, T0)
    assert got is not None and got[1] is None and got[3] is None


def test_the_output_layer_may_be_declared_first():
    torch.manual_seed(0)
    func = Sequential()
    got = mlp_field_of(func, _z0(), C, T0)
    assert got is not None and got[0] is func.inp[0].weight and got[2] is func.out.weight


def test_both_orderings_are_probed_when_both_fit():
    """The first ordering (declaration order) fails the probe, the second passes and is the one cached."""
    torch.manual_seed(0)
    func = Square()
    got = mlp_field_of(func, _z0(), 1, T0)
    assert got is not None and got[0] is func.second.weight and got[2] is func.first.weight
    assert mlp_field._recognised[func] == {True: 1}


def test_modules_with_mode_or_state_are_rejected():
    """A Dropout is refused in either mode, evaluated first or not: the probe only sees the mode it runs in."""
    torch.manual_seed(0)
    func = WithDropout().eval()
    assert mlp_field_of(func, _z0(), C, T0) is None
    func.train()
    assert mlp_field_of(func, _z0(), C, T0) is None


def test_the_verdict_follows_the_training_flag():
    """Evaluated first, then trained: the training-mode verdict is probed anew, not taken from the evaluation one."""
    torch.manual_seed(0)
    func = ModeDependent().eval()
    assert mlp_field_of(func, _z0(), C, T0) is not None
    func.train()
    assert mlp_field_of(func, _z0(), C, T0) is None
    func.eval()
    assert mlp_field_of(func, _z0(), C, T0) is not None
    assert mlp_field._recognised[func] == {False: 0, True: -1}


def test_a_batch_too_large_to_probe_is_not_a_verdict():
    torch.manual_seed(0)
    func = MlpField()
    big = torch.zeros(((1 << 27) // C) // H + 1, H)
    assert mlp_field_of(func, big, C, T0) is None
    assert func not in mlp_field._recognised
    assert mlp_field_of(func, _z0(), C, T0) is not None


def test_other_fields_are_rejected():
    torch.manual_seed(0)
    for name, body in REJECTED.items():
        assert mlp_field_of(_variant(body), _z0(), C, T0) is None, name


def test_a_third_layer_and_extra_parameters_are_rejected():
    class ThreeLayers(MlpField):
        def __init__(self):
            super().__init__()
            self.linear3 = torch.nn.Linear(H * C, H * C)

        def forward(self, tt, z):
            z = self.linear3(self.linear2(self.linear1(z).relu()).tanh()).tanh()
            return z.view(*z.shape[:-1], H, C)

    class ExtraParameter(MlpField):
        def __init__(self):
            super().__init__()
            self.scale = torch.nn.Parameter(torch.ones(()))

        def forward(self, tt, z):
            return super().forward(tt, z) * self.scale

    torch.manual_seed(0)
    assert mlp_field_of(ThreeLayers(), _z0(), C, T0) is None
    assert mlp_field_of(ExtraParameter(), _z0(), C, T0) is None


def test_shapes_must_fit():
    torch.manual_seed(0)
    assert mlp_field_of(MlpField(), _z0(), 5, T0) is None                    # wrong channel count
    assert mlp_field_of(MlpField(), torch.zeros(5, H + 1), C, T0) is None   # wrong hidden size
    assert mlp_field_of(lambda t, z: z, _z0(), C, T0) is None
    assert mlp_field_of(torch.nn.Linear(H, H * C), _z0(), C, T0) is None    # one layer: the linear field's business


def test_a_zero_state_at_time_zero_is_not_degenerate():
    """The probe uses random states at four times, so a field that differs only away from (t0, z0) is still caught."""
    zeros = torch.zeros(5, H)
    torch.manual_seed(0)
    assert mlp_field_of(_variant(REJECTED["depends_on_t"]), zeros, C, [0.0, 1.0]) is None
    assert mlp_field_of(MlpField(), zeros, C, [0.0, 1.0]) is not None


def test_the_outcome_is_cached_per_module():
    torch.manual_seed(0)
    func = MlpField()
    assert mlp_field_of(func, _z0(), C, T0) is not None
    assert mlp_field._recognised[func] == {True: 0}
    assert func not in linear_field._recognised
    calls = []
    original = func.forward
    func.forward = lambda *a: calls.append(1) or original(*a)
    assert mlp_field_of(func, _z0(), C, T0) is not None and calls == []
