# coding: utf-8
"""Model shapes the planner accepts beyond the golden cases and the BASELINE configurations: kernel sizes 1, 2, 4 and
8, one layer, one-layer stacks, gate halves above 512, residual / skip vectors of 1024, 128 conditioning channels, a
MoL head of 34 mixtures and a softmax head of 1024 classes; and ragged shapes -- vectors of 2 mod 4 that the block
count does not divide, heads of 3 channels (a Gaussian and a one-component MoL) and of 33 and 255 rows, kernel sizes
5, 6 and 7, conditioning widths of 1, 3 and 81.  Shared by tests/test_shape_coverage_host.py (planner,
packer and oracle without a GPU) and tests/test_shape_coverage.py (the kernel on an H100).

Every case is a seeded ``WaveNet`` with biases drawn from N(0, 0.05) (the reference initialises them to zero, so bias
handling would go untested), the log-scale biases of MoL / Gaussian heads lowered by 3 so that samples are not all
clipped to +-1 -- built as ``full_case`` in tests/test_gpu_parity.py builds the BASELINE configurations.

``ShapeCase`` carries what the packed-image interpreters of tests/test_host_packing.py and
tests/test_host_packing_v7.py read from a golden case (kw, sd, cfg, w, T, x_tf, t("c_up"), t("g_vec"),
arr["params_tf"]), with ``params_tf`` from a teacher-forced oracle run."""
import torch

from oracle import wavenet_oracle as orc

_SMALL = dict(residual_channels=32, gate_channels=64, skip_out_channels=32)
_MOL = dict(out_channels=30, scalar_input=True, output_distribution="Logistic", cin_channels=8)

CASES = {
    # no older taps at all: no rings, an empty ring table, a stream state of the feedback alone
    "k1": dict(kernel_size=1, layers=4, stacks=2, **_SMALL, **_MOL),
    # (kw-1)*RA = 2 rows: the packed older-tap quad is half filled
    "k2": dict(kernel_size=2, layers=6, stacks=2, **_SMALL, **_MOL),
    # 3 older taps = 6 rows in 2 quads; class-index feedback
    "k4_softmax": dict(kernel_size=4, layers=8, stacks=2, **_SMALL, out_channels=256, scalar_input=False),
    # 7 older taps, delays up to 7 * 512 = 3584: the rings live in global memory
    "k8_global": dict(kernel_size=8, layers=20, stacks=2, residual_channels=64, gate_channels=128,
                      skip_out_channels=64, out_channels=2, scalar_input=True, output_distribution="Normal",
                      cin_channels=8),
    # one layer: the first blob feeds the tail directly, the skip sum is the tail's alone
    "L1": dict(kernel_size=3, layers=1, stacks=1, **_SMALL, **_MOL),
    # one-layer stacks: every dilation is 1, ring delays 1 and 2
    "dil1": dict(kernel_size=3, layers=4, stacks=4, **_SMALL, **_MOL),
    # gate half 640 (the <BT,8,8> kernel above 512) and 128 conditioning channels (a fourth conditioning group)
    "eg8": dict(kernel_size=3, layers=2, stacks=1, residual_channels=128, gate_channels=1280, skip_out_channels=128,
                out_channels=30, scalar_input=True, output_distribution="Logistic", cin_channels=128),
    # the widest residual and skip vectors
    "wide_rs": dict(kernel_size=3, layers=2, stacks=1, residual_channels=1024, gate_channels=512,
                    skip_out_channels=1024, out_channels=30, scalar_input=True, output_distribution="Logistic",
                    cin_channels=80),
    # 34 mixtures: the Gumbel argmax loops over lanes
    "mol_k34": dict(kernel_size=3, layers=4, stacks=2, **_SMALL, out_channels=102, scalar_input=True,
                    output_distribution="Logistic", cin_channels=8),
    # 1024 classes: the widest second head stage, the one-hot gather and the dense softmax feedback
    "softmax_wide": dict(kernel_size=3, layers=4, stacks=2, residual_channels=64, gate_channels=128,
                         skip_out_channels=256, out_channels=1024, scalar_input=False),
    # ---- ragged shapes: residual, gate half and skip of 2 mod 4, odd heads, odd conditioning widths.  n rows over P
    # blocks are split n % P blocks of ceil(n / P) rows and the rest one row fewer (wn_plan.h wn_part), so a vector
    # that P does not divide leaves some blocks' row quads partly filled, or the blocks past n with no rows at all
    # a Gaussian head of 3 channels (mean y[1], log-scale y[2]); kernel size 5 (8 older-tap rows in 2 quads);
    # 6 blocks: 4 own 2 skip rows and 2 own one, 3 own a head row and 3 none
    "gauss3_r6": dict(kernel_size=5, layers=6, stacks=2, residual_channels=6, gate_channels=12, skip_out_channels=10,
                      out_channels=3, scalar_input=True, output_distribution="Normal", cin_channels=3),
    # a one-component MoL: the Gumbel argmax over one logit and a loss mixture of one term; one conditioning channel;
    # 10 blocks: 4 own 2 skip rows and 6 own one, 3 own a head row and 7 none
    "mol_k1": dict(kernel_size=3, layers=4, stacks=2, residual_channels=10, gate_channels=20, skip_out_channels=14,
                   out_channels=3, scalar_input=True, output_distribution="Logistic", cin_channels=1),
    # kernel size 7 (12 older-tap rows in 3 quads); 81 conditioning channels (a third group, partly filled and odd);
    # 26 blocks: 18 own a residual row and 8 none, 22 own a skip row and 4 none, 7 own 2 head rows and 19 one
    "mol_k11": dict(kernel_size=7, layers=8, stacks=2, residual_channels=18, gate_channels=52, skip_out_channels=22,
                    out_channels=33, scalar_input=True, output_distribution="Logistic", cin_channels=81),
    # 255 classes: the odd tail of the paired exchange poll at a tile of 1 (2 elements per thread); kernel size 6
    # (10 older-tap rows, the third quad half filled); stacks of 2 layers; 18 blocks: 3 own 15 head rows and 15 own
    # 14, residual 8 x 2 + 10 x 1, skip 12 x 2 + 6 x 1; 60 items at a tile of 4, just under the 64 limit
    "softmax_255": dict(kernel_size=6, layers=6, stacks=3, residual_channels=26, gate_channels=36,
                        skip_out_channels=30, out_channels=255, scalar_input=False),
}
NAMES = list(CASES)

# the largest batch each case runs at; wide_rs is refused at a batch tile of 4 (shared memory)
MAX_B = {n: (1 if n == "wide_rs" else 3) for n in NAMES}
# head-output tolerance against the oracle and against float64: the full-width configurations' bound for the wide cases
PARAM_TOL = {n: (1e-4 if n in ("eg8", "wide_rs", "softmax_wide") else 2e-5) for n in NAMES}


def full_kw(name):
    kw = dict(CASES[name], dropout=0.0)
    kw.setdefault("cin_channels", -1)
    kw.setdefault("gin_channels", -1)
    return kw


def path_config(kw):
    return orc.PathConfig(out_channels=kw["out_channels"], layers=kw["layers"], stacks=kw["stacks"],
                          residual_channels=kw["residual_channels"], gate_channels=kw["gate_channels"],
                          skip_out_channels=kw["skip_out_channels"], kernel_size=kw["kernel_size"],
                          cin_channels=kw["cin_channels"], gin_channels=kw["gin_channels"],
                          scalar_input=kw["scalar_input"],
                          output_distribution=kw.get("output_distribution", "Logistic"))


def max_delay(kw):
    """Steps between writing and reading the oldest tap of the most dilated layer."""
    return (kw["kernel_size"] - 1) * 2 ** (kw["layers"] // kw["stacks"] - 1)


def make_module(name, seed=0):
    """The seeded CPU module of a case (eval mode)."""
    from wavenet_vocoder_b200 import WaveNet
    kw = full_kw(name)
    torch.manual_seed(seed)
    m = WaveNet(**kw).eval()
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith(".bias"):
                p.normal_(0, 0.05)
        if kw["scalar_input"]:
            O = kw["out_channels"]
            b = m.last_conv_layers[3].bias
            if O == 2:
                b[1] -= 3.0
            else:
                b[2 * (O // 3):] -= 3.0
    return m


def fresh_module(kw, sd, dtype=torch.float32):
    """A new module with the case's weights.  (copy.deepcopy of a weight-normed module fails once it has run.)"""
    from wavenet_vocoder_b200 import WaveNet
    m = WaveNet(**kw)
    m.load_state_dict(sd)
    return m.to(dtype).eval()


def teacher_input(cfg, B, T, gen):
    if cfg.scalar_input:
        return (torch.rand(B, 1, T, generator=gen) * 2 - 1) * 0.8
    idx = torch.randint(0, cfg.out_channels, (B, T), generator=gen)
    return torch.zeros(B, cfg.out_channels, T).scatter_(1, idx.unsqueeze(1), 1.0)


class ShapeCase:
    """One case at batch B and length T: weights, seeded teacher-forcing input and sample-rate conditioning, and the
    oracle's teacher-forced head outputs (B,O,T)."""

    def __init__(self, name, B=1, T=48, seed=0, oracle=True):
        self.name = name
        self.kw = full_kw(name)
        self.module = make_module(name, seed)
        self.sd = {k: v.detach().clone() for k, v in self.module.state_dict().items()}
        self.cfg = path_config(self.kw)
        self.w = orc.weights_from_state_dict(self.cfg, self.sd)
        self.B, self.T = B, T
        gen = torch.Generator().manual_seed(1000 + 17 * B + T)
        self.x_tf = teacher_input(self.cfg, B, T, gen)
        self.arr = {}
        if self.cfg.cin_channels > 0:
            self.arr["c_up"] = torch.randn(B, self.cfg.cin_channels, T, generator=gen).numpy()
        if not oracle:
            return
        rec = []
        with torch.no_grad():
            orc.incremental_forward(self.cfg, self.w, test_inputs=self.x_tf, c=self.t("c_up"), T=T,
                                    softmax=False, quantize=False,
                                    noise=orc.replay_from_predrawn(self.cfg, orc.predraw_noise(self.cfg, B, T, 1)),
                                    params_out=rec)
        self.arr["params_tf"] = torch.stack(rec, dim=-1).numpy()

    def t(self, key):
        return None if key not in self.arr else torch.from_numpy(self.arr[key])

    def forward64(self):
        """Head outputs of the module's batch forward() in float64 on the same inputs (B,O,T)."""
        m = fresh_module(self.kw, self.sd, torch.float64)
        c = self.t("c_up")
        with torch.no_grad():
            return m(self.x_tf.double(), c=None if c is None else c.double(), softmax=False)
