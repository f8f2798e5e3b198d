"""s2g_face — host mirror of nets/smplx_face.py (inference): raw 16 kHz waveform -> jaw(3) +
expression(100) per 30 fps frame, through the wav2vec2-based regressor in the CUDA engine.  With convert_to_6d the
reference builds the identity-free net (identity=False) with a 6-D jaw head: jaw(6) + expression(100)."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from ..data_utils.utils import get_mfcc_ta
from .base import resolve_device, shared_engine, strip_module


_HF_TORCH_LAYERDROP = None


def hf_layerdrop_uses_torch_rng():
    """Does the installed ``transformers`` draw the wav2vec2 encoder's LayerDrop probabilities from TORCH's default CPU
    generator?  Newer releases do — ``dropout_probability = torch.rand([])`` once per encoder layer per forward, in eval
    mode too — so the reference's face pass (nets/spg/wav2vec.py:76-143 -> Wav2Vec2Encoder.forward) moves the generator
    that the PixelCNN sampler of the following body pass draws from (scripts/demo.py:173-204).  The release the reference
    pins (transformers~=4.22.1, requirements.txt:2) used ``np.random.uniform`` there and left torch's generator alone."""
    global _HF_TORCH_LAYERDROP
    if _HF_TORCH_LAYERDROP is None:
        try:
            import inspect

            from transformers.models.wav2vec2 import modeling_wav2vec2 as m

            _HF_TORCH_LAYERDROP = "torch.rand(" in inspect.getsource(m.Wav2Vec2Encoder.forward)
        except Exception:
            _HF_TORCH_LAYERDROP = False
    return _HF_TORCH_LAYERDROP


def face_gt(poses, expression):
    """__call__'s target (:107-111): poses [B,C,F] and expression [B,100,F] -> [B,F,C+100]."""
    poses, expression = poses.to(torch.float32), expression.to(torch.float32)
    if poses.dim() != 3 or expression.dim() != 3 or expression.shape[1] != 100 or poses.shape[0] != expression.shape[0] \
            or poses.shape[2] != expression.shape[2]:
        raise ValueError("face evaluate: poses %s, expression %s (expected [B,C,F] and [B,100,F])"
                         % (tuple(poses.shape), tuple(expression.shape)))
    return torch.cat([poses.permute(0, 2, 1), expression.permute(0, 2, 1)], 2)


def score_face(engine, wave, idv, gt):
    """get_loss (:139-167) of the regressor's prediction at frame = F against gt [B,F,C] ->
    ({'MSELoss', 'exp_loss'} as floats, the same two per clip as float64 tensors)."""
    B, F_ = gt.shape[:2]
    clip, _ = engine.face_score(wave, idv, gt)
    clip = clip.cpu()
    per_clip = {"MSELoss": clip[:, 0] / (F_ * 6), "exp_loss": clip[:, 1] / (F_ * 100)}
    return {"MSELoss": float(clip[:, 0].sum() / (B * F_ * 6)), "exp_loss": float(clip[:, 1].sum() / (B * F_ * 100))}, per_clip


class TrainWrapper:
    # torch.rand([]) draws consumed from the default CPU generator per forward, so that a seeded run of the demo flow samples
    # the same body codes as the reference does in the same environment.  None: what the reference would consume with the
    # installed transformers (one per encoder layer if hf_layerdrop_uses_torch_rng(), else 0); an int forces it (0 = the
    # behaviour of the pinned transformers 4.22.1).  The regressor itself is deterministic either way.
    layerdrop_rng_draws = None

    def __init__(self, args, config, engine=None):
        self.args = args
        self.config = config
        self.device = resolve_device(self.args.gpu)
        self.convert_to_6d = self.config.Data.pose.convert_to_6d
        self.expression = self.config.Data.pose.expression
        self.num_classes = 4
        # nets/smplx_face.py:63-93 (init_params, scale 2 for 6-D); the 6-D net has no id_mlp (:37-45, identity=False)
        if self.convert_to_6d:
            self.each_dim = [6, 144, 180, 100 if self.expression else 0]
            self.dim_list = [0, 6, 18, 150, 330]
        else:
            self.each_dim = [3, 75, 90, 100 if self.expression else 0]
            self.dim_list = [0, 3, 9, 75, 165]
        self.engine = engine or shared_engine(self.device)

    def load_state_dict(self, state_dict):
        """ckpt['generator'] of a face checkpoint: {'generator': Generator sd, ...} (nets/base.py:38-54).  Like the
        reference's strict load, a checkpoint whose output geometry is not the config's raises RuntimeError."""
        sd = strip_module(state_dict["generator"] if "generator" in state_dict else state_dict)
        got = [int(sd[k].shape[0]) if k in sd else 0 for k in ("final_out.0.weight", "final_out.1.weight")]
        identity = "audio_middle.id_mlp.weight" in sd
        if got != [self.each_dim[0], self.each_dim[3]] or identity == self.convert_to_6d:
            raise RuntimeError("s2g_face: the checkpoint's net (jaw %d + expression %d columns, %s) is not the one the config "
                               "builds (convert_to_6d=%s: jaw %d + expression %d, %s)"
                               % (got[0], got[1], "id_mlp" if identity else "identity-free", self.convert_to_6d,
                                  self.each_dim[0], self.each_dim[3], "identity-free" if self.convert_to_6d else "id_mlp"))
        self._loaded = sd
        self.engine.load_face(self._loaded)
        self.encoder_layers = len({k.split(".")[3] for k in self._loaded if k.startswith("audio_encoder.encoder.layers.")})

    def state_dict(self):
        """nets/base.py:29-36: {'generator': ..., optimizer / discriminator slots empty}."""
        return {"generator": getattr(self, "_loaded", None), "generator_optim": None, "discriminator": None,
                "discriminator_optim": None}

    def evaluate(self, bat):
        """The forward half of the reference's training step __call__(bat) (:95-167) in eval mode.  bat: 'aud_feat'
        [B,1,N] (the 16 kHz waveform; permuted and flattened to [B,N] as :106 does), 'poses' [B,C,F], 'expression'
        [B,100,F], 'speaker' [B] (id = one_hot(speaker - 20)).  Returns (None, {'MSELoss', 'exp_loss'}); per-clip values
        are kept as self.last_losses.  Kept from the reference, on purpose:
          - 'MSELoss' is an L1 over the first 6 columns in both geometries (on the 3-D net: the jaw and the first three
            expression columns of the prediction, against the first 6 columns of poses);
          - the reference sets time_steps = F only in training mode; the regressor runs with frame = F here;
          - 'grad' is not reported: there is no backward pass.
        It consumes the same torch.rand([]) draws as generate_ids."""
        if not self.expression:
            raise NotImplementedError("the face regressor is built with its expression head (config/face.json)")
        aud = torch.as_tensor(bat["aud_feat"]).to(torch.float32)
        wave = aud.permute(0, 2, 1).reshape(aud.shape[0], -1)
        gt = face_gt(torch.as_tensor(bat["poses"]), torch.as_tensor(bat["expression"]))
        if gt.shape[0] != wave.shape[0]:
            raise ValueError("face evaluate: %d waveforms for %d pose clips" % (wave.shape[0], gt.shape[0]))
        idv = F.one_hot((torch.as_tensor(bat["speaker"]) - 20).reshape(-1).to(torch.int64), self.num_classes).to(torch.float32)
        self._mirror_reference_rng()
        losses, self.last_losses = score_face(self.engine, wave, idv, gt)
        return None, losses

    def infer_on_audio(self, aud_fn, id=None, initial_pose=None, norm_stats=None, w_pre=False, frame=None, am=None,
                       am_sr=16000, **kwargs):
        """wav path or tensor [B,1,N] -> numpy (B, frame, 103), (B, frame, 106) with convert_to_6d (nets/smplx_face.py:169-218)."""
        if self.config.Data.pose.normalization:
            raise NotImplementedError("normalised face outputs are outside the built path (config/face.json: false)")
        B = 1 if initial_pose is None else initial_pose.shape[0]
        if torch.is_tensor(aud_fn):
            wave = aud_fn.to(torch.float32).reshape(aud_fn.shape[0], -1)
        else:
            feat = get_mfcc_ta(aud_fn, am=am if am is not None else True, am_sr=am_sr, fps=30,
                               encoder_choice="faceformer")                    # (N,1)
            wave = torch.from_numpy(feat[:, 0].copy())[None].repeat(B, 1)
        if frame is None:
            frame = wave.shape[1] * 30 // 16000
        if id is None:
            idv = torch.zeros(1, self.num_classes)
        else:
            idv = F.one_hot(id.reshape(-1).to(torch.int64), self.num_classes).to(torch.float32)
        return self.generate_ids(wave, idv, frame).cpu().numpy()

    def _mirror_reference_rng(self):
        n = self.layerdrop_rng_draws
        if n is None:
            n = getattr(self, "encoder_layers", 0) if hf_layerdrop_uses_torch_rng() else 0
        for _ in range(int(n)):
            torch.rand([])

    def generate_ids(self, wave, idv, frame):
        self._mirror_reference_rng()
        return self.engine.face_forward(wave, idv, frame)

    def generate(self, wv2_feat, frame):
        """tensor API (:221-238): wv2_feat [B,1,N] -> torch (B, frame, 103 or 106); id = zeros."""
        wave = wv2_feat.to(torch.float32).reshape(wv2_feat.shape[0], -1)
        return self.generate_ids(wave, torch.zeros(wave.shape[0], self.num_classes), frame)
