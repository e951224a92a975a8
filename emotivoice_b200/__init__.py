"""emotivoice_b200 -- H100-native engine for EmotiVoice's JETSGenerator.forward()
(PromptTTS acoustic model + HiFi-GAN generator).  See DESIGN.md."""
__version__ = "0.1.0"
