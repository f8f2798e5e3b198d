"""TEST INFRASTRUCTURE: the convert_to_6d pieces of the CPU oracle, built on oracle/talkshow_oracle.py's restatements.

  face_forward       s2g_face.Generator.forward for either geometry, read from the state dict: with
                     ``audio_middle.id_mlp.*`` the identity net (talkshow_oracle.face_forward), without it the identity-free
                     net of convert_to_6d configs (nets/spg/s2g_face.py:107-139, identity=False): no id columns, and
                     first_net layer 0 is relu(LN(conv(x)) + x) (nets/layers.py:95-96, in == out -> nn.Identity).
  assemble_pose_6d   scripts/demo.py:185-229 for one sample of a convert_to_6d config.
  body_vq_roundtrip_6d / body_vq_continuity_6d
                     s2g_body_vq.infer_on_audio over the 6-D pose layout (nets/smplx_body_vq.py:96-126, 208-295).
Never imported by the package."""
import torch
import torch.nn.functional as F

import talkshow_oracle as O
from talkshow_b200.data_utils.lower_body import c_index_6d


def face_forward(sd, wave, id_onehot, frame):
    """wave [B,N], id_onehot [B,4] (ignored by the identity-free net) -> [B,frame,jaw+100]."""
    if "audio_middle.id_mlp.weight" in sd:
        return O.face_forward(sd, wave, id_onehot, frame)
    h = O.wav2vec2(sd, "audio_encoder.", wave, frame)
    x = F.linear(h, sd["audio_feature_map.weight"], sd["audio_feature_map.bias"]).transpose(1, 2)
    f = "audio_middle.first_net.conv_layers."
    for i in range(3):
        x = O._cnr_ln(sd, f + "%d." % i, x, "id")
    outs = []
    for b in range(2):
        m = x
        for i in range(3):
            m = O._cnr_ln(sd, "decoder.%d.%d." % (b, i), m)
        outs.append(F.conv1d(m, sd["final_out.%d.weight" % b], sd["final_out.%d.bias" % b]))
    return torch.cat(outs, 1).transpose(1, 2)


def assemble_pose_6d(face, body, stand=False):
    """face [Ff,106] (6-D jaw | expression), body [Fb,258] (43 joints x 6-D) -> [Ff,265]: jaw and body to axis-angle,
    body padded with its last frame / truncated to Ff, cat[jaw | body | expression] -> part2full."""
    n = face.shape[0]
    jaw = O.rot6d_to_axis_angle(face[:, :6])
    if body.shape[0] < n:
        body = torch.cat([body, body[-1:].repeat(n - body.shape[0], 1)], 0)
    else:
        body = body[:n]
    body = O.rot6d_to_axis_angle(body.reshape(n, -1, 6)).reshape(n, -1)
    return O.part2full(torch.cat([jaw, body, face[:, 6:]], -1), stand)


def body_vq_roundtrip_6d(vq_ckpt, initial_pose):
    """initial_pose [B,330,F] -> (idx_body [B,T], idx_hand [B,T], numpy-layout [F, B*258])."""
    gt = initial_pose[:, c_index_6d].permute(0, 2, 1)
    ib, rb = O.vq_roundtrip(vq_ckpt["g_body"], gt[..., :78])
    ih, rh = O.vq_roundtrip(vq_ckpt["g_hand"], gt[..., 78:])
    pred = torch.cat([rb, rh], 1).transpose(1, 2)
    return ib, ih, torch.cat(list(pred), 1)


def body_vq_continuity_6d(vq_ckpt, initial_pose, chunk=60, nchunks=5):
    """continuity=True: five 60-frame chunks round-tripped on their own, concatenated in time -> [5*60, B*258]."""
    gt = initial_pose[:, c_index_6d].permute(0, 2, 1)
    bs, hs = [], []
    for i in range(nchunks):
        seg = gt[:, i * chunk:(i + 1) * chunk]
        bs.append(O.vq_roundtrip(vq_ckpt["g_body"], seg[..., :78])[1])
        hs.append(O.vq_roundtrip(vq_ckpt["g_hand"], seg[..., 78:])[1])
    pred = torch.cat([torch.cat(bs, 2), torch.cat(hs, 2)], 1).transpose(1, 2)
    return torch.cat(list(pred), 1)
