"""Native vocoders behind the reference's registry/dispatch surface
(models/vocoders/vocoder_inference.py:39-75)."""
from .apnet import APNet, ISTFT, ISTFTHead
from .bigvgan import BigVGAN
from .diffwave import DiffWave
from . import diffusion_vocoder_inference
from .hifigan import HiFiGAN, HiFiGAN_vits
from .melgan import MelGAN
from .nsfhifigan import NSFHiFiGAN
from .vocos import Vocos
from .facodec import FACodecDecoder, FACodecDecoderV2, FACodecEncoder, FACodecEncoderV2, FACodecRedecoder
from .amphion_codec import CodecDecoder, CodecEncoder
from .repcodec import RepCodec
from .gan_vocoder_inference import synthesis_audios, synthesize_to_files
from .gan_vocoder_inference import vocoder_inference as _gan_vocoder_inference

# same shape as the reference's registries: generator name -> class / functions
_vocoders = {"hifigan": HiFiGAN, "bigvgan": BigVGAN, "nsfhifigan": NSFHiFiGAN, "melgan": MelGAN, "apnet": APNet}
_vocoder_forward_funcs = {k: _gan_vocoder_inference for k in _vocoders}
_vocoder_infer_funcs = {k: synthesis_audios for k in _vocoders}
_vocoders["diffwave"] = DiffWave
_vocoder_forward_funcs["diffwave"] = diffusion_vocoder_inference.vocoder_inference
_vocoder_infer_funcs["diffwave"] = diffusion_vocoder_inference.synthesis_audios

# Vocos, the FACodec classes, the codec's CodecEncoder / CodecDecoder and RepCodec are not in the registry: the reference has no entry for them, and their constructors take
# keyword arguments, not cfg
__all__ = ["HiFiGAN", "HiFiGAN_vits", "BigVGAN", "DiffWave", "NSFHiFiGAN", "MelGAN", "APNet", "Vocos", "FACodecDecoder", "FACodecEncoder", "FACodecRedecoder", "FACodecEncoderV2", "FACodecDecoderV2", "CodecEncoder", "CodecDecoder", "RepCodec", "ISTFT", "ISTFTHead", "synthesis_audios", "synthesize_to_files", "_vocoders",
           "_vocoder_forward_funcs", "_vocoder_infer_funcs"]

# `amphion_b200.vocoders.vocoder_inference` is the MODULE (synthesis, load_nnvocoder), as
# models/vocoders/vocoder_inference.py is in the reference; the function of that name lives where the reference keeps
# it, in gan_vocoder_inference (models/vocoders/gan/gan_vocoder_inference.py:11).  Loading the submodule here makes the
# package attribute the module from the start instead of flipping when somebody first imports it.
from . import vocoder_inference  # noqa: E402,F401
from .vocoder_inference import load_nnvocoder, synthesis  # noqa: E402

__all__ += ["load_nnvocoder", "synthesis", "vocoder_inference"]
