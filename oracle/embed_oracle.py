"""Oracle of LSeg's normalised pixel embedding: `image_features` of modules/models/lseg_net.py:185-191 (head1, then
each pixel's out_c-vector divided by its L2 norm), restated with the reference's own ops and layout, as fp32 NCHW."""
import torch.nn.functional as F


def image_features(path_1, sd):
    """path_1 fp32 [B,256,h,w] (the decoder output, oracle.lseg_oracle.decoder) -> fp32 NCHW [B,out_c,h,w]."""
    f = F.conv2d(path_1, sd["scratch.head1.weight"], sd["scratch.head1.bias"])
    imshape = f.shape
    rows = f.permute(0, 2, 3, 1).reshape(-1, imshape[1])
    rows = rows / rows.norm(dim=-1, keepdim=True)
    return rows.view(imshape[0], imshape[2], imshape[3], imshape[1]).permute(0, 3, 1, 2).contiguous()
