"""Whisper's language codes in token order (<|en|> = lang_first): the 99 of the 51865-token vocabulary, then <|yue|>,
the 100th, which only the 51866-token vocabulary of the large-v3 family has.  Equivalent of the table WIS keeps in
wis/languages.py:3-103; the order is fixed by the multilingual tokenizer."""
LANGUAGE_CODES = (
    "en zh de es ru ko fr ja pt tr pl ca nl ar sv it id hi fi vi he uk el ms cs ro da hu ta no th ur hr bg lt la mi ml "
    "cy sk te fa lv bn sr az sl kn et mk br eu is hy ne mn bs kk sq sw gl mr pa si km sn yo so af oc ka be tg sd gu am "
    "yi lo uz fo ht ps tk nn mt sa lb my bo tl mg as tt haw ln ha ba jw su yue"
).split()
assert len(LANGUAGE_CODES) == 100
