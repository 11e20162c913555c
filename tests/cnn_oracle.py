"""``oracle.net.OracleNet`` with the reference's DownsampleCNN stem (models.py:278-297), in the same functional torch (fp32, or
fp64 through ``dtype``): conv(k = 2 ceil(H/16), stride 4, pad 2) + ReLU + maxpool(3, 2), conv(5, pad 2) + ReLU +
maxpool(3, 2), adaptive average to the hidden board."""
import torch.nn.functional as F

from oracle.net import OracleNet


class CnnOracleNet(OracleNet):
    def _downsample(self, p, x):
        if self.spec.downsample != 2:
            return super()._downsample(p, x)
        w = self.w
        x = F.max_pool2d(F.relu(F.conv2d(x, w[f"{p}.features.0.weight"], w[f"{p}.features.0.bias"], 4, 2)), 3, 2)
        x = F.max_pool2d(F.relu(F.conv2d(x, w[f"{p}.features.3.weight"], w[f"{p}.features.3.bias"], 1, 2)), 3, 2)
        return F.adaptive_avg_pool2d(x, self.spec.hidden_hw)
