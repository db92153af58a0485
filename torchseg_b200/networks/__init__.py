from .bisenet import BiSeNet, SpatialPath, BiSeNetHead
from .fcn import FCN
from .pspnet import PSPNet, PyramidPooling
from .dfn import DFN, DFNHead
from .psanet import PSANet, PointwiseSpatialAttention
from .deeplabv3plus import DeepLabV3Plus, ASPP, Decoder
from .encnet import EncNet, EncModule, EncHead
from .ocnet import OCNet
from .denseaspp import DenseASPP
from .danet import DANet, DANetHead
from .ocrnet import OCRNet
