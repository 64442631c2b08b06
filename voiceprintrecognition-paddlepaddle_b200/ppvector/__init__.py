"""ppvector -- H100-native drop-in for the hot path of yeyupiaoling/VoiceprintRecognition-PaddlePaddle.

Same Python surface as the reference package (``ppvector.data_utils.featurizer.AudioFeaturizer``,
``ppvector.models.build_model``, ``ppvector.predict.PPVectorPredictor``, ``ppvector.trainer.PPVectorTrainer``);
tensors are ``torch`` CUDA tensors and every hot-path op is a call into ``libppv_b200.so``
(hand-written sm_90a CUDA behind a C ABI, ``include/ppv_b200.h``).  There is no CPU fallback.
"""
__version__ = "1.1.1+b200.0"
