"""Name= -> component chain factory (reference: common/model_builder.py:26-184, :273-319).

Only the branches on the accelerated path are built: encoders `gcn_diag` (DiagGcn layers), `compgcn` (CompGcn layers,
which the reference does not have; they learn the relation codes), `gcn_basis` (BasisGcn, or ConcatGcn
when Concatenation=Yes, BasisGcnTimesDiag when DiagonalCoefficients=Yes; with UseInputTransform=No layer 0 is a one-hot
BasisGcn; SkipConnections=Highway wraps every
feature-input layer in a HighwayLayer), `embedding`, and the variational encoders `variational_embedding` and
`variational_gcn_basis` (a VariationalEncoding over two linear AffineTransform heads); decoders `bilinear-diag`, `complex`,
`rotate` (RotatE, which the reference does not have), `transe` (TransE, L1 distance; nor this), `quate` (QuatE,
quaternion rotations; nor this, with all three training objectives), `hole` (HolE, circular correlation; nor this, with
all three training objectives) and `conve` (ConvE, 1-N training only).  Unknown names return None exactly
like the reference (:270, :320); ablation flags that select out-of-scope variants raise."""
from ..decoders.bilinear_diag import BilinearDiag, parse_training_objective
from ..decoders.complex import Complex
from ..decoders.conve import ConvE
from ..decoders.hole import HolE
from ..decoders.quate import QuatE
from ..decoders.rotate import Rotate
from ..decoders.transe import TransE
from ..encoders.affine_transform import AffineTransform
from ..encoders.message_gcns.gcn_basis import BasisGcn
from ..encoders.message_gcns.gcn_basis_concat import ConcatGcn
from ..encoders.message_gcns.gcn_basis_times_diag import BasisGcnTimesDiag
from ..encoders.message_gcns.compgcn import CompGcn, parse_composition
from ..encoders.message_gcns.gcn_diag import DiagGcn
from ..encoders.relation_embedding import RelationEmbedding
from ..extras.graph_representations import Representation
from ..extras.highway_layer import HighwayLayer
from ..extras.variational_encoding import VariationalEncoding


def _flag(settings, key, default="No"):
    return settings[key] if key in settings else default


def build_encoder(encoder_settings, triples):
    name = encoder_settings['Name']
    if name == "embedding":
        input_shape = [int(encoder_settings['EntityCount']), int(encoder_settings['CodeDimension'])]
        embedding = AffineTransform(input_shape, encoder_settings, onehot_input=True, use_bias=False,
                                    use_nonlinearity=False)
        return RelationEmbedding(input_shape, encoder_settings, next_component=embedding)

    if name == "gcn_diag":
        # model_builder.py:71-119: always an input AffineTransform, then NumberOfLayers DiagGcn layers (the last one
        # linear), the optional output projection and RelationEmbedding.  The branch reads none of
        # UseInputTransform, SkipConnections, Concatenation, DiagonalCoefficients, AddDiagonal, StoreEdgeData or
        # RandomInput, so neither does this one.
        graph = Representation(triples, encoder_settings)
        d_int = int(encoder_settings['InternalEncoderDimension'])
        input_shape = [int(encoder_settings['EntityCount']), d_int]
        internal_shape = [d_int, d_int]
        projection_shape = [d_int, int(encoder_settings['CodeDimension'])]
        relation_shape = [int(encoder_settings['EntityCount']), int(encoder_settings['CodeDimension'])]
        layers = int(encoder_settings['NumberOfLayers'])
        encoding = AffineTransform(input_shape, encoder_settings, next_component=graph, onehot_input=True,
                                   use_bias=True, use_nonlinearity=True)
        for layer in range(layers):
            encoding = DiagGcn(internal_shape, encoder_settings, next_component=encoding, onehot_input=False,
                               use_nonlinearity=layer < layers - 1)
        if _flag(encoder_settings, 'UseOutputTransform') == "Yes":
            encoding = AffineTransform(projection_shape, encoder_settings, next_component=encoding,
                                       onehot_input=False, use_nonlinearity=False, use_bias=True)
        return RelationEmbedding(relation_shape, encoder_settings, next_component=encoding)

    if name == "compgcn":
        # A bias-free linear one-hot embedding of width InternalEncoderDimension, then NumberOfLayers CompGcn layers
        # (the last one linear, of width CodeDimension).  The relation codes are the top layer's Z^L[0:R]: no
        # RelationEmbedding and no output projection, since the relation codes would not pass through one.  The basis
        # and ablation flags are not read.
        parse_composition(encoder_settings)
        if _flag(encoder_settings, 'UseOutputTransform') == "Yes":
            raise ValueError("Encoder Name=compgcn takes no UseOutputTransform=Yes: the relation codes would not "
                             "pass through the output projection")
        skip = _flag(encoder_settings, 'SkipConnections', 'None')
        if skip != 'None':
            raise ValueError("Encoder Name=compgcn takes no SkipConnections (got %r): the relation codes would not "
                             "pass through them" % skip)
        graph = Representation(triples, encoder_settings)
        d_int = int(encoder_settings['InternalEncoderDimension'])
        d_code = int(encoder_settings['CodeDimension'])
        layers = int(encoder_settings['NumberOfLayers'])
        if layers < 1:
            raise ValueError("Encoder Name=compgcn needs NumberOfLayers >= 1, got %d" % layers)
        encoding = AffineTransform([int(encoder_settings['EntityCount']), d_int], encoder_settings,
                                   next_component=graph, onehot_input=True, use_bias=False, use_nonlinearity=False)
        for layer in range(layers):
            top = layer == layers - 1
            encoding = CompGcn([d_int, d_code if top else d_int], encoder_settings, next_component=encoding,
                               use_nonlinearity=not top, owns_relations=layer == 0, top=top)
        return encoding

    if name == "gcn_basis":
        graph = Representation(triples, encoder_settings)
        d_int = int(encoder_settings['InternalEncoderDimension'])
        input_shape = [int(encoder_settings['EntityCount']), d_int]
        internal_shape = [d_int, d_int]
        projection_shape = [d_int, int(encoder_settings['CodeDimension'])]
        relation_shape = [int(encoder_settings['EntityCount']), int(encoder_settings['CodeDimension'])]
        layers = int(encoder_settings['NumberOfLayers'])

        if _flag(encoder_settings, 'UseInputTransform') == "Yes":
            encoding = AffineTransform(input_shape, encoder_settings, next_component=graph, onehot_input=True,
                                       use_bias=True, use_nonlinearity=True)
        elif _flag(encoder_settings, 'RandomInput') == "Yes" or _flag(encoder_settings, 'PartiallyRandomInput') == "Yes":
            raise NotImplementedError("RandomInput / PartiallyRandomInput variants are outside the accelerated path "
                                      "(SURVEY.md 2.1 #6)")
        else:
            encoding = graph   # featureless: layer 0 reads one-hot entity input (model_builder.py:166-167)
        encoding = apply_basis_gcn(encoder_settings, encoding, internal_shape, layers)
        if _flag(encoder_settings, 'UseOutputTransform') == "Yes":
            encoding = AffineTransform(projection_shape, encoder_settings, next_component=encoding,
                                       onehot_input=False, use_nonlinearity=False, use_bias=True)
        return RelationEmbedding(relation_shape, encoder_settings, next_component=encoding)

    if name == "variational_embedding":
        # model_builder.py:43-69: two bias-free one-hot tables, mu = W_mu and log sigma = W_sigma
        input_shape = [int(encoder_settings['EntityCount']), int(encoder_settings['CodeDimension'])]
        mu = AffineTransform(input_shape, encoder_settings, onehot_input=True, use_bias=False, use_nonlinearity=False)
        sigma = AffineTransform(input_shape, encoder_settings, onehot_input=True, use_bias=False,
                                use_nonlinearity=False)
        z = VariationalEncoding(input_shape, encoder_settings, mu_network=mu, sigma_network=sigma)
        return RelationEmbedding(input_shape, encoder_settings, next_component=z)

    if name == "variational_gcn_basis":
        # model_builder.py:186-254: the gcn_basis trunk, two biased linear heads for mu and log sigma, the
        # reparameterised code, then the optional output projection and RelationEmbedding
        graph = Representation(triples, encoder_settings)
        d_int = int(encoder_settings['InternalEncoderDimension'])
        input_shape = [int(encoder_settings['EntityCount']), d_int]
        internal_shape = [d_int, d_int]
        projection_shape = [d_int, int(encoder_settings['CodeDimension'])]
        relation_shape = [int(encoder_settings['EntityCount']), int(encoder_settings['CodeDimension'])]
        layers = int(encoder_settings['NumberOfLayers'])
        if _flag(encoder_settings, 'UseInputTransform') == "Yes":
            encoding = AffineTransform(input_shape, encoder_settings, next_component=graph, onehot_input=True,
                                       use_bias=True, use_nonlinearity=True)
        elif _flag(encoder_settings, 'RandomInput') == "Yes" or _flag(encoder_settings, 'PartiallyRandomInput') == "Yes":
            # the branch reads neither flag (:206-214) but apply_basis_gcn does: layer 0 would be a feature layer
            # reading the graph object itself
            raise NotImplementedError("UseInputTransform=No with RandomInput / PartiallyRandomInput: the reference's "
                                      "variational_gcn_basis hands the graph object to a feature-input layer")
        else:
            encoding = graph
        encoding = apply_basis_gcn(encoder_settings, encoding, internal_shape, layers)
        mu = AffineTransform(projection_shape, encoder_settings, next_component=encoding, onehot_input=False,
                             use_nonlinearity=False, use_bias=True)
        sigma = AffineTransform(projection_shape, encoder_settings, next_component=encoding, onehot_input=False,
                                use_nonlinearity=False, use_bias=True)
        encoding = VariationalEncoding(input_shape, encoder_settings, mu_network=mu, sigma_network=sigma)
        if _flag(encoder_settings, 'UseOutputTransform') == "Yes":
            encoding = AffineTransform(projection_shape, encoder_settings, next_component=encoding,
                                       onehot_input=False, use_nonlinearity=False, use_bias=True)
        return RelationEmbedding(relation_shape, encoder_settings, next_component=encoding)
    return None


def apply_basis_gcn(encoder_settings, encoding, internal_shape, layers):
    # the reference's layer precedence (model_builder.py:285-294): AddDiagonal > DiagonalCoefficients > StoreEdgeData
    # > Concatenation
    diagonal_coefficients = False
    for flag in ('AddDiagonal', 'DiagonalCoefficients', 'StoreEdgeData'):
        if _flag(encoder_settings, flag) != "Yes":
            continue
        if flag == 'DiagonalCoefficients' and _flag(encoder_settings, 'UseInputTransform') != "No":
            diagonal_coefficients = True
            break
        if flag == 'DiagonalCoefficients':
            raise NotImplementedError("DiagonalCoefficients=Yes with UseInputTransform=No: the featureless first "
                                      "layer would need its own per-channel push kernel, which is not built")
        raise NotImplementedError("%s=Yes selects an ablation variant outside the accelerated path" % flag)
    skip = _flag(encoder_settings, 'SkipConnections', 'None')
    if skip not in ('None', 'Residual', 'Highway'):
        raise NotImplementedError("SkipConnections=%s is not a reference option" % skip)
    if skip == 'Highway' and _flag(encoder_settings, 'UseInputTransform') == "No":
        # In the reference, layer 1's highway reads its carry input from MessageGcn's class-level cache, which by
        # then holds layer 1's own output: out = g L1 + (1 - g) L1 = L1 and the gate gets zero gradient.  Neither
        # that dead gate nor a working one (which would silently differ from the reference) is built.
        raise NotImplementedError("SkipConnections=Highway with UseInputTransform=No: the reference's highway gate "
                                  "is dead there (its carry input is the layer's own output through the shared "
                                  "MessageGcn cache), so this combination is not built")
    if diagonal_coefficients:
        model = BasisGcnTimesDiag
    else:
        model = ConcatGcn if _flag(encoder_settings, 'Concatenation') == "Yes" else BasisGcn
    for layer in range(layers):
        use_nonlinearity = layer < layers - 1  # the last layer is linear (model_builder.py:275)
        # only layer 0 of a featureless encoder reads one-hot input (model_builder.py:277-283)
        onehot_input = (layer == 0 and _flag(encoder_settings, 'UseInputTransform') == "No"
                        and _flag(encoder_settings, 'RandomInput') == "No"
                        and _flag(encoder_settings, 'PartiallyRandomInput') == "No")
        new_encoding = model(internal_shape, encoder_settings, next_component=encoding, onehot_input=onehot_input,
                             use_nonlinearity=use_nonlinearity)
        # 'Residual' is a no-op in the reference (model_builder.py:302-307: the else branch overwrites it)
        if skip == 'Highway' and not onehot_input:
            encoding = HighwayLayer(internal_shape, next_component=new_encoding, next_component_2=encoding)
        else:
            encoding = new_encoding
    return encoding


def build_decoder(encoder, decoder_settings):
    if decoder_settings['Name'] == "conve":
        # ConvE scores every entity per query: 1-N is its only objective
        objective = parse_training_objective(decoder_settings)[0]
        if objective != '1-N':
            raise ValueError("the conve decoder trains under TrainingObjective=1-N only, not %r" % objective)
        return ConvE(int(decoder_settings['CodeDimension']), decoder_settings, next_component=encoder)
    if decoder_settings['Name'] == "quate":
        # linear in each row, as DistMult: all three objectives (NegativeSampling, SelfAdversarial, 1-N) on the same
        # scoring GEMMs; BilinearDiag.parse_settings checks the objective keys
        return QuatE(int(decoder_settings['CodeDimension']), decoder_settings, next_component=encoder)
    if decoder_settings['Name'] == "hole":
        # linear in each row once in its Fourier basis: all three objectives on the same scoring GEMMs, as QuatE
        return HolE(int(decoder_settings['CodeDimension']), decoder_settings, next_component=encoder)
    if decoder_settings['Name'] not in ("bilinear-diag", "complex"):
        objective = parse_training_objective(decoder_settings)[0]
        # RotatE and TransE train under SelfAdversarial (the objective of the RotatE paper) but have no 1-N scoring GEMM
        if objective != 'NegativeSampling' and not (decoder_settings['Name'] in ("rotate", "transe")
                                                    and objective == 'SelfAdversarial'):
            raise ValueError("TrainingObjective=%s needs the bilinear-diag or complex decoder, not %r"
                             % (objective, decoder_settings['Name']))
    if decoder_settings['Name'] == "bilinear-diag":
        return BilinearDiag(encoder, decoder_settings)
    if decoder_settings['Name'] == "complex":
        return Complex(int(decoder_settings['CodeDimension']), decoder_settings, next_component=encoder)
    if decoder_settings['Name'] == "rotate":
        return Rotate(int(decoder_settings['CodeDimension']), decoder_settings, next_component=encoder)
    if decoder_settings['Name'] == "transe":
        return TransE(int(decoder_settings['CodeDimension']), decoder_settings, next_component=encoder)
    return None
