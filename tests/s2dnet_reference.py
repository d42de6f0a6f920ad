"""S2DNet at num_layers 1, restated with torch.nn.functional for the tests (float64 by default, CPU or GPU).

The network, from the reference's model (VGG16's first four encoder layers and one adaptation layer):
    x  = (rgb / 255 - mean) / std                      ImageNet mean and std, per channel
    a1 = relu(conv2d(x, encoder.0, padding 1))
    a2 = relu(conv2d(a1, encoder.2, padding 1))
    a3 = relu(conv2d(a2, adap.0, padding 0))           1 x 1
    f  = batch_norm(conv2d(a3, adap.2, padding 2))     5 x 5, eval mode, eps 1e-5, no ReLU after it
    out = f / max(||f||, 1e-12) over the 128 channels  when l2_normalize
Every convolution pads its own input with zeros.  `write_checkpoint` writes seeded weights under the reference's key
names, plus keys of deeper layers that a num_layers 1 model ignores."""
import numpy as np

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
ADAP = "adaptation_layers.adap_layer_0."


def seeded_state_dict(seed=0, extra=True):
    """kaiming-normal convolutions, random biases and BatchNorm statistics (float32 tensors, as a checkpoint holds)"""
    import torch
    g = torch.Generator().manual_seed(seed)

    def conv(cout, cin, k):
        w = torch.empty(cout, cin, k, k)
        std = (2.0 / (cin * k * k)) ** 0.5                     # kaiming normal, fan_in, ReLU gain
        return w.normal_(0, std, generator=g), torch.empty(cout).uniform_(-0.1, 0.1, generator=g)

    sd = {}
    sd["encoder.0.weight"], sd["encoder.0.bias"] = conv(64, 3, 3)
    sd["encoder.2.weight"], sd["encoder.2.bias"] = conv(64, 64, 3)
    sd[ADAP + "0.weight"], sd[ADAP + "0.bias"] = conv(64, 64, 1)
    sd[ADAP + "2.weight"], sd[ADAP + "2.bias"] = conv(128, 64, 5)
    sd[ADAP + "3.weight"] = torch.empty(128).uniform_(0.5, 1.5, generator=g)
    sd[ADAP + "3.bias"] = torch.empty(128).uniform_(-0.2, 0.2, generator=g)
    sd[ADAP + "3.running_mean"] = torch.empty(128).uniform_(-0.5, 0.5, generator=g)
    sd[ADAP + "3.running_var"] = torch.empty(128).uniform_(0.5, 2.0, generator=g)
    if extra:
        sd[ADAP + "3.num_batches_tracked"] = torch.tensor(1000)
        sd["encoder.5.weight"], sd["encoder.5.bias"] = conv(128, 64, 3)
        sd["adaptation_layers.adap_layer_1.0.weight"], sd["adaptation_layers.adap_layer_1.0.bias"] = conv(64, 256, 1)
    return sd


def write_checkpoint(path, seed=0, state_dict=None):
    """a file torch.load(path, weights_only=True)["state_dict"] reads back"""
    import torch
    torch.save({"state_dict": state_dict if state_dict is not None else seeded_state_dict(seed)}, str(path))
    return path


def forward(image, state_dict, l2_normalize=True, dtype=None, device="cpu"):
    """[H, W, 3] uint8 -> [H, W, 128] map (a torch tensor of `dtype`, float64 by default)"""
    import torch
    import torch.nn.functional as Fn
    dtype = dtype or torch.float64
    p = {k: v.to(device=device, dtype=dtype) for k, v in state_dict.items() if v.is_floating_point()}
    image = image if torch.is_tensor(image) else torch.from_numpy(np.ascontiguousarray(image))
    x = image.to(device).permute(2, 0, 1)[None].to(dtype) / 255
    x = (x - torch.tensor(MEAN, dtype=dtype, device=device)[:, None, None]) / \
        torch.tensor(STD, dtype=dtype, device=device)[:, None, None]
    x = Fn.relu(Fn.conv2d(x, p["encoder.0.weight"], p["encoder.0.bias"], padding=1))
    x = Fn.relu(Fn.conv2d(x, p["encoder.2.weight"], p["encoder.2.bias"], padding=1))
    x = Fn.relu(Fn.conv2d(x, p[ADAP + "0.weight"], p[ADAP + "0.bias"]))
    x = Fn.conv2d(x, p[ADAP + "2.weight"], p[ADAP + "2.bias"], padding=2)
    x = Fn.batch_norm(x, p[ADAP + "3.running_mean"], p[ADAP + "3.running_var"], p[ADAP + "3.weight"], p[ADAP + "3.bias"],
                      training=False, eps=1e-5)
    if l2_normalize:
        x = Fn.normalize(x, dim=1)
    return x[0].permute(1, 2, 0)
